"""The opt-in FP8 (e4m3) self-attention: the fused RMSNorm+RoPE quantiser and the V^T pre-pass bit for bit against their
torch restatements, attention_fp8 against the fp32 oracle next to a restated fp8 chain, the whole model against the fp32
oracle with that chain in its self-attention, and the model-level guarantees (toggling off, determinism, CUDA graphs, the
cross-K/V cache, context parallelism refused, bad ABI arguments refused).  TF32 is off throughout."""
import math

import pytest
import torch

from test_fp8_gpu import SMALL, deq, lib_fp8_linear, quant_ref, rel, rnd, small_inputs
from test_scale_gpu import sdpa_fp32_chunked

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn
# the key stored at V^T column k inside each 16-key group: the order of P's e4m3 A fragment (written out, not computed)
PI16 = [0, 1, 8, 9, 2, 3, 10, 11, 4, 5, 12, 13, 6, 7, 14, 15]


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def pad(L):
    return (L + 127) // 128 * 128


def qk_ref(x, B, H, L):
    """Q or K bf16 [B*L, H*128] -> (codes [B*L, H*128], head-major scales [B, H, L_pad] zero past L) by quant_ref per head."""
    q, s = quant_ref(x.reshape(-1, 128))
    sp = torch.zeros(B, H, pad(L), device=x.device)
    sp[:, :, :L] = s.view(B, L, H).permute(0, 2, 1)
    return q.view(B * L, H * 128), sp


def vt_ref(v, B, H, L):
    """V bf16 [B*L, H*128] -> (V^T codes [B, H, 128, L_pad] in the kernel's key order, zero past L; scales [B, H, 128])."""
    rows = v.view(B, L, H, 128).permute(0, 2, 3, 1).reshape(B * H * 128, L)
    q, s = quant_ref(rows)
    q = q.view(torch.uint8).view(B, H, 128, L)
    Lp = pad(L)
    full = torch.zeros(B, H, 128, Lp, device=v.device, dtype=torch.uint8)
    full[..., :L] = q
    perm = torch.tensor([16 * (k // 16) + PI16[k % 16] for k in range(Lp)], device=v.device)
    return full[..., perm], s.view(B, H, 128)


# ---------------------------------------------------------------- 1. RMSNorm + RoPE, fp8 form
@pytest.mark.parametrize("B,L,H", [(2, 1000, 2), (1, 130, 3), (2, 27904, 40)])
def test_rmsnorm_rope_fp8_bit_exact(B, L, H):
    from scail_b200 import ops
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=L)
    wq, wk = rnd(d, seed=1) + 1, rnd(d, seed=2) + 1
    wq[128:256] = 0  # head 1 of every Q row is all zero: scale 1, codes 0
    ang = torch.rand(L, 128, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda") * 6.3
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()  # per-token tables: any values exercise the RoPE path
    before = qkv.clone()
    Lp = pad(L)
    q8 = (torch.empty(B * L, d, device="cuda", dtype=FP8), torch.full((B, H, Lp), 7.0, device="cuda"))
    k8 = (torch.empty(B * L, d, device="cuda", dtype=FP8), torch.full((B, H, Lp), 7.0, device="cuda"))
    ops.rmsnorm_rope(qkv, L, d, [(0, wq), (d, wk)], cos, sin, out_fp8=[q8, k8])
    assert torch.equal(qkv, before)  # the fp8 form reads the buffer only
    ref = before.clone()
    ops.rmsnorm_rope(ref, L, d, [(0, wq), (d, wk)], cos, sin)
    for (q, s), col in ((q8, 0), (k8, d)):
        qr, sr = qk_ref(ref[:, col:col + d], B, H, L)
        assert torch.equal(s, sr)
        assert torch.equal(q.view(torch.uint8), qr.view(torch.uint8))
    # the zero head (w = 0 gives +-0): scale 1, codes +-0
    assert float(q8[1][0, 1, 0]) == 1.0 and not (q8[0][:, 128:256].view(torch.uint8) & 0x7F).any()


# ---------------------------------------------------------------- 2. V^T pre-pass
@pytest.mark.parametrize("L,H", [(64, 2), (130, 2), (1000, 3), (48832, 40)])
def test_quant_vt_bit_exact(L, H):
    from scail_b200 import ops
    B, d = 2, H * 128
    qkv = rnd(B * L, 3 * d, seed=L + 1)
    qkv[:L, 2 * d + 5] = 0  # batch 0, head 0, channel 5: an all-zero channel
    qkv[3, 2 * d + 7] = 1.0e4  # one large outlier
    v = qkv[:, 2 * d:]  # the V column slab of the fused buffer, ldv = 3 d
    vt = torch.full((B, H, 128, pad(L)), 0x7F, device="cuda", dtype=torch.uint8).view(FP8)  # NaN everywhere before
    sc = torch.empty(B, H, 128, device="cuda")
    ops.quant_vt_fp8(v, B, H, L, vt, sc)
    want, ws = vt_ref(v, B, H, L)
    assert torch.equal(sc, ws)
    assert torch.equal(vt.view(torch.uint8), want)
    assert float(sc[0, 0, 5]) == 1.0 and not vt.view(torch.uint8)[0, 0, 5].any()
    key = torch.tensor([16 * (k // 16) + PI16[k % 16] for k in range(pad(L))], device="cuda")
    assert not vt.view(torch.uint8)[..., key >= L].any()  # the padding keys are zero


# ---------------------------------------------------------------- 3. the kernel
def chain_fp8(q, k, v, chunk=256):
    """The restated fp8 chain in fp32 ([B, H, L, 128] inputs): dequantised Q^, K^ (per token and head), V^ (per channel),
    P^ = e4m3(2^8 p) against the final row max, l the sum of the unquantised 2^8 p."""
    B, H, L, D = q.shape
    qd = deq(*quant_ref(q.reshape(-1, D))).view(B, H, L, D)
    kd = deq(*quant_ref(k.reshape(-1, D))).view(B, H, L, D)
    vtr = v.transpose(-1, -2).reshape(-1, L)
    vd = deq(*quant_ref(vtr)).view(B, H, D, L).transpose(-1, -2)
    out = torch.empty(B, H, L, D, device=q.device)
    kt = kd.transpose(-1, -2)
    for i in range(0, L, chunk):
        s = (qd[:, :, i:i + chunk] @ kt) * D ** -0.5
        p = torch.exp(s - s.amax(-1, keepdim=True)) * 256.0
        out[:, :, i:i + chunk] = (p.to(FP8).float() @ vd) / p.sum(-1, keepdim=True)
        del s, p
    return out


@pytest.mark.parametrize("B,H,L", [(1, 2, 256), (2, 2, 1000), (2, 3, 64), (2, 40, 27904)])
def test_attention_fp8_against_fp32_and_chain(B, H, L):
    from scail_b200 import ops
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=B * L + H)
    # one query row whose top logit dominates (a key in the last tile): P^ = 2^8 there, ~0 elsewhere
    qkv[5, :128] = 4.0 * qkv[L - 3, d:d + 128].float().to(torch.bfloat16)
    q4 = qkv.view(B, L, 3, H, 128)
    qh, kh, vh = (q4[:, :, i].transpose(1, 2).float() for i in range(3))
    q8, qs = qk_ref(qkv[:, :d], B, H, L)
    k8, ks = qk_ref(qkv[:, d:2 * d], B, H, L)
    vt, vs = ops.quant_vt_fp8(qkv[:, 2 * d:], B, H, L)
    out = torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16)
    ops.attention_fp8(q8, qs, k8, ks, vt, vs, out, B, H, L)
    torch.cuda.synchronize()
    want = sdpa_fp32_chunked(qh, kh, vh, 512).transpose(1, 2).reshape(B * L, d)
    chain = chain_fp8(qh, kh, vh).transpose(1, 2).reshape(B * L, d)
    assert torch.isfinite(out.float()).all()
    e, e_chain = rel(out, want), rel(chain, want)
    print(f"attention_fp8 B={B} H={H} L={L}: ours vs fp32 {e:.3e} | restated fp8 chain vs fp32 {e_chain:.3e} | "
          f"ours vs chain {rel(out, chain):.3e}")
    assert e <= 1.25 * e_chain + 1e-3, (e, e_chain)
    e_row = rel(out[5, :128], chain[5, :128])  # the whole weight on one key: P^ = 2^8 there in both
    assert e_row < 1e-2, e_row


# ---------------------------------------------------------------- 4. the model against the fp32 oracle
def small_model(seed=0, **kw):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(seed)
    m = DiffusionTransformer(**SMALL, **kw).to(torch.bfloat16).cuda().eval()
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    return m


def oracle_with_fp8_chain(O, args, linears):
    """O.dit_forward with the restated fp8 chain as the self-attention sdpa (q_len == kv_len; cross-attention keeps the
    oracle's fp32 sdpa) and, with `linears`, the library FP8 chain for the six per-block linears."""
    from test_fp8_gpu import SIX
    old_sdpa, old_lin = O.sdpa, O.linear

    def sdpa(q, k, v):
        if q.shape[-2] == k.shape[-2]:
            return chain_fp8(q.float(), k.float(), v.float())
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


def oracle_fp32(O, args):
    old = O.sdpa
    O.sdpa = lambda q, k, v: sdpa_fp32_chunked(q, k, v) if q.dtype == torch.float32 else old(q, k, v)
    try:
        with torch.no_grad(), torch.device("cuda"):
            return O.dit_forward(*args)
    finally:
        O.sdpa = old


def check_model(what, m, x, kw, args):
    """Ours with fp8 attention (alone, then with fp8 linears) against the fp32 oracle, next to the oracle with the restated
    fp8 chain.  That chain rounds nothing to bf16 outside the ops it restates, while ours does everywhere; so the bound adds
    our bf16 forward's error (measured on the same model) in quadrature to the chain's: 1.25 * hypot(chain, bf16) + 1e-3."""
    import oracle.dit_oracle as O
    ad = m.mixins["adaln_layer"]
    want = oracle_fp32(O, args)
    for linears in (False, True):
        ad.fp8_attention, ad.fp8_linear = True, linears
        with torch.no_grad():
            got = m(x, **kw).float()
        ad.fp8_attention = ad.fp8_linear = False
        with torch.no_grad():
            got16 = m(x, **kw).float()
        chain = oracle_with_fp8_chain(O, args, linears)
        e, e_chain, e16 = rel(got, want), rel(chain, want), rel(got16, want)
        mode = "fp8 attention + fp8 linears" if linears else "fp8 attention"
        print(f"{what}, {mode}, vs fp32 oracle: ours {e:.3e} | restated fp8 chain {e_chain:.3e} | ours bf16 {e16:.3e}")
        assert e <= 1.25 * math.hypot(e_chain, e16) + 1e-3, (mode, e, e_chain, e16)


def test_small_model_against_oracle():
    m = small_model(3)
    x, kw = small_inputs(4)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), kw["timesteps"], kw["context"].float(), kw["ref_concat"].float(),
            kw["concat_smpl_render"].float(), kw["image_clip_features"].float(), 2, 2)
    check_model("small 2-layer model", m, x, kw, args)


def test_full_width_block_at_config_A_against_oracle():
    """One 14B-width block (5120 / 40 heads / 13824) at N = 27 904, b = 1, as test_fp8_gpu.py."""
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(3)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            m = DiffusionTransformer(hidden_size=5120, num_attention_heads=40, inner_hidden_size=13824, num_layers=1,
                                     text_dim=4096, time_embed_dim=5120).eval()
    finally:
        torch.set_default_dtype(prev)
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    g = torch.Generator().manual_seed(6)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    b, t, h, w = 1, 21, 64, 64
    x, ref, pose = r(b, t, 16, h, w), r(1, 1, 16, h, w), r(1, t, 16, h // 2, w // 2)
    ctx, clip, ts = r(b, 512, 4096), r(1, 257, 1280), torch.tensor([500.0]).cuda()
    kw = dict(timesteps=ts, context=ctx, ref_concat=ref, concat_smpl_render=pose, image_clip_features=clip, concat_images=x)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), ts, ctx.float(), ref.float(), pose.float(), clip.float(), 40, 1)
    check_model("config-A block (N=27904, b=1)", m, x, kw, args)


# ---------------------------------------------------------------- 5. model-level guarantees
def test_toggle_off_reproduces_bf16_and_fp8_forward_is_deterministic():
    x, kw = small_inputs(5)
    never = small_model(6)
    m = small_model(6, fp8_attention=True)
    with torch.no_grad():
        want = never(x, **kw).clone()
        on = m(x, **kw).clone()
        again = m(x, **kw).clone()
        m.mixins["adaln_layer"].fp8_attention = False
        off = m(x, **kw).clone()
    assert torch.equal(off, want)
    assert not torch.equal(on, want)
    assert torch.equal(on, again)
    sa, sb = m.state_dict(), never.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.parametrize("fp8_linear", [False, True])
def test_graphed_step_and_cross_kv_cache_bit_identical(fp8_linear):
    from scail_b200 import sampler
    m = small_model(15, fp8_attention=True, fp8_linear=fp8_linear)
    g = torch.Generator().manual_seed(2)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
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


def test_context_parallel_refused():
    class StubCP:
        size, rank = 2, 0

    m = small_model(1, fp8_attention=True)
    m.mixins["adaln_layer"].cp = StubCP()
    x, kw = small_inputs(2)
    with pytest.raises(NotImplementedError, match="fp8_attention"), torch.no_grad():
        m(x, **kw)


# ---------------------------------------------------------------- 6. the ABI refuses bad arguments
def test_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    h = _lib.lib()
    B, H, L, Lp = 1, 2, 200, 256
    q8 = torch.zeros(B * L, H * 128, device="cuda", dtype=torch.uint8)
    sc = torch.ones(B, H, Lp, device="cuda")
    vt = torch.zeros(B, H, 128, Lp, device="cuda", dtype=torch.uint8)
    vs = torch.ones(B, H, 128, device="cuda")
    out = torch.empty(B * L, H * 128, device="cuda", dtype=torch.bfloat16)
    P = lambda t: t.data_ptr()

    def att(**kw):
        a = dict(Q=P(q8), ldq=H * 128, qs=P(sc), K=P(q8), ldk=H * 128, ks=P(sc), vt=P(vt), vs=P(vs), out=P(out), ldo=H * 128,
                 B=B, H=H, hd=128, L=L, Lp=Lp)
        a.update(kw)
        rc = h.scail_attention_fp8(*a.values(), 0.088, None)
        return rc, h.scail_last_error()

    rc, err = att()
    assert rc == 0, err
    torch.cuda.synchronize()
    for kw, msg in [(dict(hd=64), b"head_dim"), (dict(L=300), b"L <= L_pad"), (dict(Lp=200), b"L_pad"),
                    (dict(ldq=H * 128 + 8), b"multiples of 16"), (dict(K=None), b"null operand"),
                    (dict(Q=P(q8) + 8), b"16-byte aligned")]:
        rc, err = att(**kw)
        assert rc == -1 and msg in err, (kw, err)
    v = torch.zeros(B * L, H * 128, device="cuda", dtype=torch.bfloat16)
    work = torch.empty(B, H * 128, device="cuda", dtype=torch.int32)
    rc = h.scail_quant_vt_fp8(P(v), H * 128, P(vt), P(vs), P(work), B, H, 64, L, Lp, None)
    assert rc == -1 and b"head_dim" in h.scail_last_error()
    rc = h.scail_quant_vt_fp8(P(v), H * 128, P(vt), P(vs), None, B, H, 128, L, Lp, None)
    assert rc == -1 and b"null operand" in h.scail_last_error()
    w = torch.ones(192, device="cuda", dtype=torch.bfloat16)
    buf = torch.zeros(L, 3 * 192, device="cuda", dtype=torch.bfloat16)
    rc = h.scail_rmsnorm_rope_fp8(P(buf), 3 * 192, L, L, 192, 1, 0, P(w), 0, None, None, None, 1e-6, P(q8), P(sc), None, None,
                                  192, Lp, None)
    assert rc == -1 and b"multiple of the 128-wide head" in h.scail_last_error()
