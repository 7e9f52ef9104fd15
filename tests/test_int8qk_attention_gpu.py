"""fp8_attention="int8_qk": INT8 Q and smoothed INT8 K, e4m3 V and P.

1. The quantisers bit for bit against a torch restatement of the INT8 row format (restated below), in row-strided slabs of
   the fused QKV buffer (ld 15 360): Q and its scales, K written back in bf16, k-bar against the fp64 mean, K' from the
   kernel's own k-bar; repeat launches bit-identical.
2. The attention kernel, dense, against the fp32 softmax of the unquantised bf16 operands, next to the fp8 kernel on the same
   inputs and a restated int8-QK chain: within 1.25x of the chain overall and 2x of its worst (batch, head, 128-query)
   block, and at most 0.8x the fp8 kernel's error.
3. The sparse forms: the full map bit-identical to dense, a window map and per-(batch, head) adaptive maps within the same
   bounds against the masked fp32 softmax; the INT8 tile pooling bit for bit.
4. Smoothing against a planted per-(batch, head) channel offset in K.
5. The model against the fp32 oracle, toggling off, CUDA graphs and the cross-K/V cache.
The mode's launches of the 14B step at every geometry, b = 2 and b = 1, are checked against fp32 in
tests/test_dit_int8_b1_launch_shapes_gpu.py.
TF32 is off throughout."""
import math

import pytest
import torch

from test_fp8_attention_gpu import oracle_fp32, pad, qk_ref, small_model
from test_fp8_gpu import SIX, lib_fp8_linear, rel, rnd, small_inputs
from test_scale_gpu import sdpa_fp32_chunked

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn
BF = torch.bfloat16


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


# ---------------------------------------------------------------- the INT8 row format, restated
def int8_ref(x):
    """x [rows, 128] -> (codes int8, scales fp32): s = amax / 127 by IEEE division (1 for an all-zero row),
    q = round-half-even(x / s) clamped to [-127, 127].  Divisors are tensors: torch evaluates `tensor / python_float` as a
    multiplication by the reciprocal, not an IEEE division."""
    xf = x.float()
    amax = xf.abs().amax(1)
    s = torch.where(amax > 0, amax / torch.full_like(amax, 127.0), torch.ones_like(amax))
    return torch.round(xf / s[:, None]).clamp(-127, 127).to(torch.int8), s


def heads_ref(x, B, H, L):
    """Q or K' [B*L, H*128] -> (codes [B*L, H*128], head-major scales [B, H, L_pad] zero past L)."""
    q, s = int8_ref(x.reshape(-1, 128))
    sp = torch.zeros(B, H, pad(L), device=x.device)
    sp[:, :, :L] = s.view(B, L, H).permute(0, 2, 1)
    return q.view(B * L, H * 128), sp


def kbar_fp64(k, B, L):
    """The per-(batch, channel) mean over the L keys in fp64, rounded once to fp32: [B, H*128]."""
    return (k.double().view(B, L, -1).sum(1) / L).float()


def deq(q, s):
    return q.float() * s[:, None]


def ulp_f32(x):
    return (torch.nextafter(x.abs(), torch.full_like(x, math.inf)) - x.abs())


# ---------------------------------------------------------------- 1. quantisers
@pytest.mark.parametrize("L", [129, 130, 1000, 27904])
def test_quantisers_bit_exact(L):
    from scail_b200 import ops
    B, H = 2, 40
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=L)  # ld 15 360, as the fused QKV buffer
    wq, wk = rnd(d, seed=1) + 1, rnd(d, seed=2) + 1
    wq[128:256] = 0  # head 1 of every Q row is all zero: scale 1, codes 0
    ang = torch.rand(L, 128, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda") * 6.3
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    ref = qkv.clone()
    ops.rmsnorm_rope(ref, L, d, [(0, wq), (d, wk)], cos, sin)
    Lp = pad(L)
    q8 = torch.full((B * L, d), 99, device="cuda", dtype=torch.int8)
    qs = torch.full((B, H, Lp), 7.0, device="cuda")
    ops.rmsnorm_rope_int8q(qkv, L, d, [(0, wq), (d, wk)], q8, qs, cos, sin)
    qr, sr = heads_ref(ref[:, :d], B, H, L)
    assert torch.equal(qs, sr)
    assert torch.equal(q8, qr)
    assert float(qs[0, 1, 0]) == 1.0 and not q8[:, 128:256].any()
    assert torch.equal(qkv[:, d:], ref[:, d:])  # K written back in bf16 exactly as the bf16 form; V untouched
    assert torch.equal(qkv[:, :d], rnd(B * L, 3 * d, seed=L)[:, :d])  # the Q slab is read only

    k = qkv[:, d:2 * d]
    k8 = torch.full((B * L, d), 99, device="cuda", dtype=torch.int8)
    ks = torch.full((B, H, Lp), 7.0, device="cuda")
    kbar = torch.empty(B, d, device="cuda")
    ops.quant_k_int8(k, B, H, L, k8, ks, kbar)
    want_bar = kbar_fp64(k, B, L)
    assert ((kbar - want_bar).abs() <= ulp_f32(want_bar)).all(), float((kbar - want_bar).abs().max())
    kp = (k.float().view(B, L, d) - kbar[:, None, :]).view(B * L, d)  # one fp32 subtraction per element
    kr, ksr = heads_ref(kp, B, H, L)
    assert torch.equal(ks, ksr)
    assert torch.equal(k8, kr)
    again = [torch.empty_like(t) for t in (k8, ks, kbar)]
    ops.quant_k_int8(k, B, H, L, *again)
    for a, b in zip(again, (k8, ks, kbar)):
        assert torch.equal(a, b)
    print(f"L={L}: k-bar within one fp32 ulp of the fp64 mean, max |diff| {float((kbar - want_bar).abs().max()):.3g}")


# ---------------------------------------------------------------- 2. the kernel, dense
def operands(qkv, B, H, L):
    """Every operand of both kernels from one bf16 QKV buffer: the INT8 path from our quantisers (pinned bit for bit above),
    the e4m3 path from its own restatement; plus the fp32 [B, H, L, 128] views of the bf16 Q, K, V."""
    from scail_b200 import ops
    d = H * 128
    q4 = qkv.view(B, L, 3, H, 128)
    qh, kh, vh = (q4[:, :, i].transpose(1, 2).float() for i in range(3))
    qi, qis = heads_ref(qkv[:, :d], B, H, L)
    ki, kis, kbar = ops.quant_k_int8(qkv[:, d:2 * d], B, H, L)
    q8, qs = qk_ref(qkv[:, :d], B, H, L)
    k8, ks = qk_ref(qkv[:, d:2 * d], B, H, L)
    vt, vs = ops.quant_vt_fp8(qkv[:, 2 * d:], B, H, L)
    return dict(qh=qh, kh=kh, vh=vh, i8=(qi, qis, ki, kis), f8=(q8, qs, k8, ks), v=(vt, vs), kbar=kbar)


def chain_int8(q, k, v, mask=None, smooth=True, chunk=256):
    """The restated int8-QK chain in fp32 ([B, H, L, 128] inputs): dequantised INT8 Q^ and K'^ (K' = K - its fp64 per-channel
    mean when smooth), V^ per channel in e4m3, P^ = e4m3(2^8 p) against the final row max, l the sum of the unquantised
    2^8 p.  mask: optional bool [B, H, L, L] of the keys each query attends to."""
    B, H, L, D = q.shape
    qd = deq(*int8_ref(q.reshape(-1, D))).view(B, H, L, D)
    kk = k - (k.double().mean(2, keepdim=True).float() if smooth else 0.0)
    kd = deq(*int8_ref(kk.reshape(-1, D))).view(B, H, L, D)
    vtr = v.transpose(-1, -2).reshape(-1, L)
    amax = vtr.abs().amax(1)
    vsc = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
    vd = ((vtr / vsc[:, None]).clamp(-448, 448).to(FP8).float() * vsc[:, None]).view(B, H, D, L).transpose(-1, -2)
    out = torch.empty(B, H, L, D, device=q.device)
    kt = kd.transpose(-1, -2)
    for i in range(0, L, chunk):
        s = (qd[:, :, i:i + chunk] @ kt) * D ** -0.5
        if mask is not None:
            s.masked_fill_(~mask[:, :, i:i + chunk], -math.inf)
        p = torch.exp(s - s.amax(-1, keepdim=True)) * 256.0
        out[:, :, i:i + chunk] = (p.to(FP8).float() @ vd) / p.sum(-1, keepdim=True)
        del s, p
    return out


def sdpa_masked(q, k, v, mask=None, chunk=512):
    if mask is None:
        return sdpa_fp32_chunked(q, k, v, chunk)
    out = torch.empty_like(q)
    kt = k.transpose(-1, -2)
    for i in range(0, q.shape[-2], chunk):
        s = (q[..., i:i + chunk, :] @ kt) * q.shape[-1] ** -0.5
        out[..., i:i + chunk, :] = torch.softmax(s.masked_fill_(~mask[:, :, i:i + chunk], -math.inf), -1) @ v
    return out


def worst_block(got, want, B, H, L):
    """The largest rel-L2 over the (batch, head, 128-query) blocks; got, want [B*L, H*128]."""
    n = -(-L // 128)
    d = torch.nn.functional.pad((got.float() - want).pow(2).view(B, L, H, 128).sum(-1), (0, 0, 0, n * 128 - L))
    w = torch.nn.functional.pad(want.pow(2).view(B, L, H, 128).sum(-1), (0, 0, 0, n * 128 - L))
    return float((d.view(B, n, 128, H).sum(2) / w.view(B, n, 128, H).sum(2)).sqrt().max())


def merged(x, B, H, L):
    return x.transpose(1, 2).reshape(B * L, H * 128)


def verdict(out, out8, want, chain, B, H, L, what):
    e, e8, ec = rel(out, want), rel(out8, want), rel(chain, want)
    wb, wbc = worst_block(out, want, B, H, L), worst_block(chain, want, B, H, L)
    print(f"{what} B={B} H={H} L={L}: int8_qk vs fp32 {e:.3e} | fp8 kernel {e8:.3e} (ratio {e / e8:.3f}) | restated int8 "
          f"chain {ec:.3e} | worst block {wb:.3e} vs chain's {wbc:.3e}")
    assert torch.isfinite(out.float()).all()
    # The format estimate was 0.35x the fp8 kernel's error.  The restated chain itself measures 0.71-0.73x on this data: the
    # e4m3 P^ and V^, which both modes share, carry about as much of the error as Q and K did.  So the kernel is held to
    # its chain, and to a clear margin below the fp8 kernel.
    assert e <= 0.8 * e8, (e, e8)
    assert e <= 1.25 * ec, (e, ec)
    assert wb <= 2.0 * wbc, (wb, wbc)


def planted(B, H, L, seed):
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=seed)
    # one query row whose top logit dominates (a key in the last tile): P^ = 2^8 there, ~0 elsewhere
    qkv[5, :128] = 4.0 * qkv[L - 3, d:d + 128].float().to(BF)
    return qkv


@pytest.mark.parametrize("B,H,L", [(1, 2, 129), (2, 8, 1000), (2, 40, 27904)])
def test_attention_dense_against_fp32_fp8_and_chain(B, H, L):
    from scail_b200 import ops
    qkv = planted(B, H, L, B * L + H)
    o = operands(qkv, B, H, L)
    out = torch.empty(B * L, H * 128, device="cuda", dtype=BF)
    out8 = torch.empty_like(out)
    ops.attention_int8qk(*o["i8"], *o["v"], out, B, H, L)
    ops.attention_fp8(*o["f8"], *o["v"], out8, B, H, L)
    want = merged(sdpa_fp32_chunked(o["qh"], o["kh"], o["vh"], 512), B, H, L)
    chain = merged(chain_int8(o["qh"], o["kh"], o["vh"]), B, H, L)
    verdict(out, out8, want, chain, B, H, L, "dense")
    again = torch.empty_like(out)
    ops.attention_int8qk(*o["i8"], *o["v"], again, B, H, L)
    assert torch.equal(out, again)


# ---------------------------------------------------------------- 3. sparse
def tile_mask(maps, B, H, L):
    """bool [B, H, L, L] from {(b, h): (ptr, idx)} host maps (or one (ptr, idx) for every (b, h))."""
    n = -(-L // 128)
    m = torch.zeros(B, H, n, n, dtype=torch.bool)
    for b in range(B):
        for h in range(H):
            ptr, idx = maps[(b, h)] if isinstance(maps, dict) else maps
            for t in range(n):
                m[b, h, t, torch.as_tensor(idx[ptr[t]:ptr[t + 1]], dtype=torch.long)] = True
    return m.cuda().repeat_interleave(128, 2).repeat_interleave(128, 3)[:, :, :L, :L]


def test_sparse_forms():
    from scail_b200 import ops, sparse
    B, H, L = 2, 8, 1000
    n = -(-L // 128)
    qkv = planted(B, H, L, 77)
    o = operands(qkv, B, H, L)
    out = torch.empty(B * L, H * 128, device="cuda", dtype=BF)
    ops.attention_int8qk(*o["i8"], *o["v"], out, B, H, L)
    # the full map is the dense kernel
    full = ops.TileMap([n * t for t in range(n + 1)], [k for _ in range(n) for k in range(n)], L, L, device="cuda")
    got = torch.empty_like(out)
    ops.attention_int8qk(*o["i8"], *o["v"], got, B, H, L, tiles=full)
    assert torch.equal(got, out)
    # a window-1 map (tile 0 holds the reference tokens) and the per-(batch, head) adaptive maps on the INT8 operands
    ptr, idx = [0], []
    for t in range(n):
        idx += sorted({0} | {k for k in (t - 1, t, t + 1) if 0 <= k < n})
        ptr.append(len(idx))
    win = ops.TileMap(ptr, idx, L, L, device="cuda")
    qi, qis, ki, kis = o["i8"]
    ws = {}
    bh = sparse.AdaptiveTiles(0.6, 3).select(qi, ki, B, H, L, 100, lambda nm, sh, dt: ws.setdefault(nm, torch.empty(
        sh, device="cuda", dtype=dt)), q_scale=qis, k_scale=kis)
    host = sparse.bh_maps_host(*bh)
    assert any(len(i) < n * n for _, i in host.values())  # some tiles were dropped
    for what, kw, mask in (("window 1", dict(tiles=win), tile_mask((ptr, idx), B, H, L)),
                           ("adaptive", dict(bh_maps=bh), tile_mask(host, B, H, L))):
        o8 = torch.empty_like(out)
        if what == "adaptive":
            ops.attention_fp8_sparse_bh(*o["f8"], *o["v"], o8, B, H, L, *bh)
        else:
            ops.attention_fp8(*o["f8"], *o["v"], o8, B, H, L, tiles=win)
        ops.attention_int8qk(*o["i8"], *o["v"], got, B, H, L, **kw)
        want = merged(sdpa_masked(o["qh"], o["kh"], o["vh"], mask), B, H, L)
        chain = merged(chain_int8(o["qh"], o["kh"], o["vh"], mask), B, H, L)
        verdict(got, o8, want, chain, B, H, L, what)


def test_tile_pool_int8_bit_exact():
    from scail_b200 import ops
    B, H, L = 2, 3, 1000
    qkv = planted(B, H, L, 5)
    qi, qis = heads_ref(qkv[:, :H * 128], B, H, L)
    got = ops.tile_pool(qi, B, H, L, x_scale=qis)
    n = -(-L // 128)
    x = (qi.double().view(B, L, H, 128) * qis[:, :, :L].double().permute(0, 2, 1)[..., None]).permute(0, 2, 1, 3)
    want = torch.empty(B, H, n, 128, device="cuda")
    for t in range(n):  # each row's product is exact in fp64, so the sum's order does not matter
        want[:, :, t] = x[:, :, 128 * t:128 * t + 128].mean(2).float()
    assert torch.equal(got, want)


# ---------------------------------------------------------------- 4. smoothing pays for itself
def test_smoothing_absorbs_a_planted_channel_offset():
    from scail_b200 import ops
    B, H, L = 2, 4, 1000
    d = H * 128
    base = planted(B, H, L, 31)
    g = torch.Generator(device="cuda").manual_seed(4)
    off = 16.0 * torch.randn(B, 1, d, generator=g, device="cuda")  # per (batch, head, channel), the same for every key
    shifted = base.clone()
    shifted.view(B, L, 3 * d)[:, :, d:2 * d] = (base.view(B, L, 3 * d)[:, :, d:2 * d].float() + off).to(BF)
    errs = {}
    for what, qkv in (("plain", base), ("offset", shifted)):
        o = operands(qkv, B, H, L)
        out = torch.empty(B * L, d, device="cuda", dtype=BF)
        ops.attention_int8qk(*o["i8"], *o["v"], out, B, H, L)
        want = merged(sdpa_fp32_chunked(o["qh"], o["kh"], o["vh"], 512), B, H, L)
        raw = merged(chain_int8(o["qh"], o["kh"], o["vh"], smooth=False), B, H, L)
        errs[what] = (rel(out, want), rel(raw, want))
    print(f"int8_qk vs fp32: {errs['plain'][0]:.3e} without the offset, {errs['offset'][0]:.3e} with it | int8 chain without "
          f"smoothing: {errs['plain'][1]:.3e} / {errs['offset'][1]:.3e}")
    assert errs["offset"][1] >= 2.0 * errs["plain"][1], errs  # the offset matters to an unsmoothed INT8 K
    assert errs["offset"][0] <= 1.2 * errs["plain"][0], errs


# ---------------------------------------------------------------- 5. the model
def oracle_with_int8_chain(O, args, linears=False):
    """O.dit_forward with the restated int8-QK chain as the self-attention sdpa (cross-attention keeps fp32) and, with
    `linears`, the library fp8 chain for the six per-block linears."""
    old_sdpa, old_lin = O.sdpa, O.linear

    def sdpa(q, k, v):
        if q.shape[-2] == k.shape[-2]:
            return chain_int8(q.float(), k.float(), v.float())
        return sdpa_fp32_chunked(q, k, v) if q.dtype == torch.float32 else old_sdpa(q, k, v)

    def linear(sd, prefix, x):
        if prefix.startswith("transformer.layers.") and prefix.split(".", 3)[3] in SIX:
            return lib_fp8_linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))
        return old_lin(sd, prefix, x)

    O.sdpa = sdpa
    if linears:
        O.linear = linear
    try:
        with torch.no_grad(), torch.device("cuda"):
            return O.dit_forward(*args)
    finally:
        O.sdpa, O.linear = old_sdpa, old_lin


def check_model(what, m, x, kw, args):
    """int8_qk against the fp32 oracle next to the oracle with the restated chain; the bound adds our bf16 forward's error in
    quadrature, as the fp8 test does: 1.25 * hypot(chain, bf16) + 1e-3.  bf16 and fp8 are printed beside it."""
    import oracle.dit_oracle as O
    ad = m.mixins["adaln_layer"]
    want = oracle_fp32(O, args)
    res = {}
    for mode in (False, True, "int8_qk"):
        ad.fp8_attention = mode
        with torch.no_grad():
            res[mode] = rel(m(x, **kw).float(), want)
    ad.fp8_attention = False
    e_chain = rel(oracle_with_int8_chain(O, args), want)
    print(f"{what} vs fp32 oracle: int8_qk {res['int8_qk']:.3e} | fp8 {res[True]:.3e} | bf16 {res[False]:.3e} | oracle with "
          f"the int8 chain {e_chain:.3e}")
    assert res["int8_qk"] <= 1.25 * math.hypot(e_chain, res[False]) + 1e-3, res


def test_small_model_against_oracle():
    m = small_model(3)
    x, kw = small_inputs(4)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), kw["timesteps"], kw["context"].float(), kw["ref_concat"].float(),
            kw["concat_smpl_render"].float(), kw["image_clip_features"].float(), 2, 2)
    check_model("small 2-layer model", m, x, kw, args)


def full_width_model(num_layers, seed=3):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(seed)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF)
    try:
        with torch.device("cuda"):
            m = DiffusionTransformer(hidden_size=5120, num_attention_heads=40, inner_hidden_size=13824, num_layers=num_layers,
                                     text_dim=4096, time_embed_dim=5120).eval()
    finally:
        torch.set_default_dtype(prev)
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    return m


def test_full_width_block_at_config_A_against_oracle():
    """One 14B-width block (5120 / 40 heads / 13824) at N = 27 904, b = 1."""
    m = full_width_model(1)
    g = torch.Generator().manual_seed(6)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    b, t, h, w = 1, 21, 64, 64
    x, ref, pose = r(b, t, 16, h, w), r(1, 1, 16, h, w), r(1, t, 16, h // 2, w // 2)
    ctx, clip, ts = r(b, 512, 4096), r(1, 257, 1280), torch.tensor([500.0]).cuda()
    kw = dict(timesteps=ts, context=ctx, ref_concat=ref, concat_smpl_render=pose, image_clip_features=clip, concat_images=x)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), ts, ctx.float(), ref.float(), pose.float(), clip.float(), 40, 1)
    check_model("config-A block (N=27904, b=1)", m, x, kw, args)


def test_toggle_off_reproduces_bf16_and_the_mode_is_deterministic():
    x, kw = small_inputs(5)
    never = small_model(6)
    m = small_model(6, fp8_attention="int8_qk")
    with torch.no_grad():
        want = never(x, **kw).clone()
        on = m(x, **kw).clone()
        again = m(x, **kw).clone()
        m.mixins["adaln_layer"].fp8_attention = True
        fp8 = m(x, **kw).clone()
        m.mixins["adaln_layer"].fp8_attention = False
        off = m(x, **kw).clone()
    assert torch.equal(off, want)
    assert not torch.equal(on, want) and not torch.equal(on, fp8)
    assert torch.equal(on, again)


@pytest.mark.parametrize("extra", [dict(), dict(fp8_linear=True), dict(attention_window=1)], ids=["alone", "fp8_linear", "window"])
def test_graphed_step_and_cross_kv_cache_bit_identical(extra):
    from scail_b200 import sampler
    m = small_model(15, fp8_attention="int8_qk", **extra)
    g = torch.Generator().manual_seed(2)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    x0 = torch.randn(1, 3, 16, 8, 8, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, 8, 8), concat_smpl_render=r(1, 3, 16, 4, 4),
                image_clip_features=r(1, 257, 1280))
    uc = dict(crossattn=r(1, 24, 64))
    sig = sampler.make_flow_timesteps(50, 5.0)
    with torch.no_grad():
        xe = x0.clone()
        for i in range(3):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0)
        xg = x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0)
        for i in range(3):
            gs(sig[i], sig[i + 1])
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=2)
        m.mixins["adaln_layer"].cache_cross_kv = True
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=2)
    torch.cuda.synchronize()
    assert torch.equal(xe, xg)
    assert torch.equal(plain, cached)


def test_adaptive_graphed_step_bit_identical():
    from scail_b200 import sampler, sparse
    m = small_model(16, fp8_attention="int8_qk", attention_adaptive=sparse.AdaptiveTiles(0.5, 1))
    g = torch.Generator().manual_seed(3)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    x0 = torch.randn(1, 5, 16, 16, 16, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, 16, 16), concat_smpl_render=r(1, 5, 16, 8, 8),
                image_clip_features=r(1, 257, 1280))
    uc = dict(crossattn=r(1, 24, 64))
    sig = sampler.make_flow_timesteps(50, 5.0)
    with torch.no_grad():
        xe = x0.clone()
        for i in range(2):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0)
        xg = x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0)
        for i in range(2):
            gs(sig[i], sig[i + 1])
    torch.cuda.synchronize()
    assert torch.equal(xe, xg)


# ---------------------------------------------------------------- the ABI refuses bad arguments
def test_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    h = _lib.lib()
    B, H, L, Lp = 1, 2, 200, 256
    q8 = torch.zeros(B * L, H * 128, device="cuda", dtype=torch.int8)
    sc = torch.ones(B, H, Lp, device="cuda")
    vt = torch.zeros(B, H, 128, Lp, device="cuda", dtype=torch.uint8)
    vs = torch.ones(B, H, 128, device="cuda")
    out = torch.empty(B * L, H * 128, device="cuda", dtype=BF)
    ptr = torch.zeros(B, H, 3, device="cuda", dtype=torch.int32)
    P = lambda t: t.data_ptr()

    def att(**kw):
        a = dict(Q=P(q8), ldq=H * 128, qs=P(sc), K=P(q8), ldk=H * 128, ks=P(sc), vt=P(vt), vs=P(vs), out=P(out), ldo=H * 128,
                 B=B, H=H, hd=128, L=L, Lp=Lp, scale=0.088, ptr=None, ps=0, idx=None, ids=0)
        a.update(kw)
        rc = h.scail_attention_int8qk(*a.values(), None)
        return rc, h.scail_last_error()

    rc, err = att()
    assert rc == 0, err
    torch.cuda.synchronize()
    for kw, msg in [(dict(hd=64), b"head_dim"), (dict(L=300), b"L <= L_pad"), (dict(ldq=H * 128 + 8), b"multiples of 16"),
                    (dict(K=None), b"null operand"), (dict(Q=P(q8) + 8), b"16-byte aligned"),
                    (dict(ptr=P(ptr)), b"come together"), (dict(ptr=P(ptr), idx=P(ptr), ps=3), b"both 0"),
                    (dict(ptr=P(ptr), idx=P(ptr), ps=2, ids=4), b"ptr_stride")]:
        rc, err = att(**kw)
        assert rc == -1 and msg in err and b"attention_int8qk" in err, (kw, err)
    kb = torch.empty(B, H * 128, device="cuda")
    part = torch.empty(B * H * 128, device="cuda", dtype=torch.float64)
    kk = torch.zeros(B * L, H * 128, device="cuda", dtype=BF)
    rc = h.scail_quant_k_int8(P(kk), H * 128, P(q8), H * 128, P(sc), P(kb), P(part), part.numel(), B, H, L, Lp, None)
    assert rc == 0, h.scail_last_error()
    torch.cuda.synchronize()
    rc = h.scail_quant_k_int8(P(kk), H * 128, P(q8), H * 128, P(sc), P(kb), P(part), part.numel() - 1, B, H, L, Lp, None)
    assert rc == -1 and b"partial_len" in h.scail_last_error()
    rc = h.scail_quant_k_int8(P(kk), H * 128, P(q8), H * 128, P(sc), P(kb), None, 0, B, H, L, Lp, None)
    assert rc == -1 and b"null operand" in h.scail_last_error()
    buf = torch.zeros(L, 3 * H * 128, device="cuda", dtype=BF)
    w = torch.ones(H * 128, device="cuda", dtype=BF)
    rc = h.scail_rmsnorm_rope_int8q(P(buf), 3 * H * 128, L, L, H * 128, 1, 0, P(w), 0, None, None, None, 1e-6, P(q8), P(sc),
                                    H * 128, Lp, None)
    assert rc == -1 and b"nslabs" in h.scail_last_error()
    rc = h.scail_attention_tile_pool_int8(P(q8), H * 128, None, P(kb), B, H, L, Lp, None)
    assert rc == -1 and b"null operand" in h.scail_last_error()
    rc = h.scail_attention_tile_pool_int8(P(q8), H * 128, P(sc), P(kb), B, H, L, 300, None)
    assert rc == -1 and b"L_pad" in h.scail_last_error()
