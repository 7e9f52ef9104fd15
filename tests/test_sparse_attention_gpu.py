"""Block-sparse self-attention on the GPU: the sparse forms of the bf16 and fp8 kernels against the dense kernels (full map,
bit for bit), against the fp32 masked softmax (frame-window maps and maps that stress the warpgroup turns), and the model
surface (attention_window) against the masked fp32 oracle, with the guarantees of the other opt-in modes: toggling off,
determinism, CUDA graphs, the cross-K/V cache, context parallelism refused, bad ABI arguments refused.  TF32 is off."""
import math

import numpy as np
import pytest
import torch

from kernel_check import assert_close_bf16
from sparse_oracle import masked_sdpa_fp32, tile_mask
from test_fp8_attention_gpu import qk_ref
from test_fp8_gpu import SMALL, deq, quant_ref, rel, rnd

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def full_map(L):
    n = -(-L // 128)
    return np.arange(0, n * n + 1, n), np.tile(np.arange(n), n)


def masked_chain_fp8(q, k, v, mask, chunk=256):
    """chain_fp8 (test_fp8_attention_gpu.py) with the mask applied: the same dequantised operands, P^ against the row max
    over the allowed keys, masked keys contribute nothing."""
    B, H, L, D = q.shape
    qd = deq(*quant_ref(q.reshape(-1, D))).view(B, H, L, D)
    kd = deq(*quant_ref(k.reshape(-1, D))).view(B, H, L, D)
    vd = deq(*quant_ref(v.transpose(-1, -2).reshape(-1, L))).view(B, H, D, L).transpose(-1, -2)
    out = torch.empty(B, H, L, D, device=q.device)
    kt = kd.transpose(-1, -2)
    for i in range(0, L, chunk):
        s = ((qd[:, :, i:i + chunk] @ kt) * D ** -0.5).masked_fill_(~mask[i:i + chunk], float("-inf"))
        p = torch.exp(s - s.amax(-1, keepdim=True)) * 256.0
        out[:, :, i:i + chunk] = (p.to(FP8).float() @ vd) / p.sum(-1, keepdim=True)
        del s, p
    return out


def fp8_operands(qkv, B, H, L):
    from scail_b200 import ops
    d = H * 128
    q8, qs = qk_ref(qkv[:, :d], B, H, L)
    k8, ks = qk_ref(qkv[:, d:2 * d], B, H, L)
    vt, vs = ops.quant_vt_fp8(qkv[:, 2 * d:], B, H, L)
    return q8, qs, k8, ks, vt, vs


def heads(x, B, L, H):
    return x.view(B, L, H, 128).transpose(1, 2).float()


# ---------------------------------------------------------------- 1. the full map is the dense kernel, bit for bit
@pytest.mark.parametrize("B,H,L", [(2, 2, 129), (2, 2, 130), (2, 3, 1000), (1, 8, 27904)])
def test_full_map_is_bit_identical_to_the_dense_kernels(B, H, L):
    from scail_b200 import ops
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=L)
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    m = ops.TileMap(*full_map(L), L, L, device="cuda")
    a, b = (torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    ops.attention(q, k, v, a, B, H, L, L)
    ops.attention_sparse(q, k, v, b, B, H, L, m)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    q8, qs, k8, ks, vt, vs = fp8_operands(qkv, B, H, L)
    ops.attention_fp8(q8, qs, k8, ks, vt, vs, a, B, H, L)
    ops.attention_fp8_sparse(q8, qs, k8, ks, vt, vs, b, B, H, L, m)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


# ---------------------------------------------------------------- 2. against the fp32 masked softmax
L_EDGE = 6 * 128 + 37  # 7 key tiles, the last holding 37 keys
EDGE_ROWS = [[6], [0], [1, 3], [0, 2, 6], [0, 1, 2, 3, 4], [2], [0, 1, 2, 3, 4, 5, 6]]  # 1, 2, 3, 5, 7 tiles; ragged-only row


def edge_map():
    return np.cumsum([0] + [len(r) for r in EDGE_ROWS]), np.concatenate(EDGE_ROWS)


def frame_map(window, t=5, h=32, w=32):
    from scail_b200 import sparse
    H, W = h // 2, w // 2
    g = sparse.geometry(H * W, t * H * W, t * (H // 2) * (W // 2), t, H, W)
    ptr, idx, density = sparse.frame_window_tiles(g, window)
    assert density < 1.0
    return ptr, idx, g.ref_length + g.seq_length + g.pose_length


CASES = {"turn edge cases": lambda: (*edge_map(), L_EDGE),
         "window 0": lambda: frame_map(0), "window 1": lambda: frame_map(1),
         "window 2 at 512x512": lambda: frame_map(2, 21, 64, 64)}


@pytest.mark.parametrize("case", list(CASES))
def test_sparse_kernels_against_the_fp32_masked_softmax(case):
    from scail_b200 import ops
    ptr, idx, L = CASES[case]()
    B, H = (1, 2) if L > 20000 else (2, 2)
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=L + 7)
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    m = ops.TileMap(ptr, idx, L, L, device="cuda")
    mask = tile_mask(ptr, idx, L, L).cuda()
    out = torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16)
    ops.attention_sparse(q, k, v, out, B, H, L, m)
    want = masked_sdpa_fp32(heads(q, B, L, H), heads(k, B, L, H), heads(v, B, L, H), mask)
    want = want.transpose(1, 2).reshape(B * L, d)
    torch.cuda.synchronize()
    # Two bf16 roundings per term (P enters PV as bf16, then the output), and each output averages hundreds to thousands of
    # keys whose values cancel: the relative slack is two roundings (2^-7) and the absolute slack one bf16 ulp of the largest
    # output (2^-8 max|want|).  A wrong or missing tile moves elements by the output's own scale, far beyond that.
    c = assert_close_bf16(out, want, f"bf16 sparse, {case}", elem_rel=2.0 ** -7, elem_abs=2.0 ** -8)
    print(f"bf16 sparse {case} (L={L}, density {m.density:.3f}): rel-L2 {c.rel_l2:.3e}, worst |d|/bound {c.worst_ratio:.3f}")
    # fp8: within the bound test_fp8_attention_gpu.py uses against the restated chain, the mask applied to both
    q8, qs, k8, ks, vt, vs = fp8_operands(qkv, B, H, L)
    ops.attention_fp8_sparse(q8, qs, k8, ks, vt, vs, out, B, H, L, m)
    chain = masked_chain_fp8(heads(q, B, L, H), heads(k, B, L, H), heads(v, B, L, H), mask).transpose(1, 2).reshape(B * L, d)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    e, e_chain = rel(out, want), rel(chain, want)
    print(f"fp8 sparse {case}: ours vs fp32 {e:.3e} | restated masked fp8 chain vs fp32 {e_chain:.3e}")
    assert e <= 1.25 * e_chain + 1e-3, (e, e_chain)


def test_repeat_sparse_launches_are_bit_identical():
    from scail_b200 import ops
    ptr, idx, L = frame_map(1)
    B, H = 2, 4
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=3)
    m = ops.TileMap(ptr, idx, L, L, device="cuda")
    outs = []
    for fp8 in (False, True):
        for _ in range(2):
            o = torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16)
            if fp8:
                q8, qs, k8, ks, vt, vs = fp8_operands(qkv, B, H, L)
                ops.attention_fp8_sparse(q8, qs, k8, ks, vt, vs, o, B, H, L, m)
            else:
                ops.attention_sparse(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], o, B, H, L, m)
            outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[2], outs[3])


# ---------------------------------------------------------------- 3. the model against the masked fp32 oracle
def small_model(seed=0, **kw):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(seed)
    m = DiffusionTransformer(**SMALL, **kw).to(torch.bfloat16).cuda().eval()
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    return m


def small_inputs(seed=1, t=5, h=32, w=32):
    """b = 2 at a latent large enough (N = 1856, 15 tiles) for window 1 to mask: frame_map(1) has density < 1."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    x, ref, pose = r(2, t, 16, h, w), r(1, 1, 16, h, w), r(1, t, 16, h // 2, w // 2)
    kw = dict(timesteps=torch.tensor([400.0, 400.0]).cuda(), context=r(2, 24, 64), ref_concat=ref, concat_smpl_render=pose,
              image_clip_features=r(1, 257, 1280), concat_images=x)
    return x, kw


def oracle(args, key_mask=None, fp8_chain=False):
    """O.dit_forward in fp32 (chunked sdpa) with the key mask on the self-attention; fp8_chain: the masked restated fp8
    chain as the self-attention instead."""
    import oracle.dit_oracle as O
    old = O.sdpa

    def sdpa(q, k, v):
        if q.dtype != torch.float32:
            return old(q, k, v)
        full = torch.ones(q.shape[-2], k.shape[-2], dtype=torch.bool, device=q.device)
        if q.shape[-2] != k.shape[-2]:  # cross-attention (24, 257 or 512 keys): never masked
            return masked_sdpa_fp32(q, k, v, full)
        mask = full if key_mask is None else key_mask
        return masked_chain_fp8(q, k, v, mask) if fp8_chain else masked_sdpa_fp32(q, k, v, mask)

    O.sdpa = sdpa
    try:
        with torch.no_grad(), torch.device("cuda"):
            return O.dit_forward(*args)
    finally:
        O.sdpa = old


def check_model(what, m, x, kw, args, window, fp8):
    """Ours with the window against the masked fp32 oracle; the bound is our dense forward's error against the unmasked
    oracle (bf16), or the fp8 model test's bound with the masked chain (fp8_attention)."""
    from scail_b200 import sparse
    ad = m.mixins["adaln_layer"]
    b, t, _, h, w = x.shape
    H, W = h // 2, w // 2
    g = sparse.geometry(H * W, t * H * W, t * (H // 2) * (W // 2), t, H, W)
    ptr, idx, density = sparse.frame_window_tiles(g, window)
    assert density < 1.0
    N = g.ref_length + g.seq_length + g.pose_length
    mask = tile_mask(ptr, idx, N, N).cuda()
    want_dense, want = oracle(args), oracle(args, mask)
    assert not torch.equal(want, want_dense)  # the mask changes the function
    with torch.no_grad():
        ad.attention_window, ad.fp8_attention = None, False
        dense16 = m(x, **kw).float()
        ad.attention_window = window
        got16 = m(x, **kw).float()
        if fp8:
            ad.fp8_attention = True
            got8 = m(x, **kw).float()
        ad.attention_window, ad.fp8_attention = None, False
    e16, e_dense = rel(got16, want), rel(dense16, want_dense)
    print(f"{what}, window {window} (density {density:.3f}): bf16 sparse vs masked oracle {e16:.3e} | dense vs oracle "
          f"{e_dense:.3e}")
    assert e16 <= 1.25 * e_dense + 1e-3, (e16, e_dense)
    if fp8:
        chain = oracle(args, mask, fp8_chain=True)
        e8, e_chain = rel(got8, want), rel(chain, want)
        print(f"{what}, window {window}, fp8_attention: ours {e8:.3e} | masked fp8 chain {e_chain:.3e} | ours bf16 {e16:.3e}")
        assert e8 <= 1.25 * math.hypot(e_chain, e16) + 1e-3, (e8, e_chain, e16)


def test_small_model_window_1_against_masked_oracle():
    m = small_model(3)
    x, kw = small_inputs(4)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), kw["timesteps"], kw["context"].float(), kw["ref_concat"].float(),
            kw["concat_smpl_render"].float(), kw["image_clip_features"].float(), 2, 2)
    check_model("small 2-layer model", m, x, kw, args, 1, fp8=True)


def test_full_width_block_at_config_A_against_masked_oracle():
    """One 14B-width block (5120 / 40 heads / 13824) at N = 27 904, b = 1, window 2."""
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
    check_model("config-A block (N=27904, b=1)", m, x, kw, args, 2, fp8=False)


# ---------------------------------------------------------------- 4. model-level guarantees
@pytest.mark.parametrize("fp8_attention", [False, True])
def test_full_window_and_toggling_off_reproduce_the_dense_forward(fp8_attention):
    x, kw = small_inputs(5)
    m = small_model(6, fp8_attention=fp8_attention)
    ad = m.mixins["adaln_layer"]
    with torch.no_grad():
        want = m(x, **kw).clone()
        ad.attention_window = x.shape[1] - 1  # T - 1: the full map, through the sparse kernel
        full = m(x, **kw).clone()
        ad.attention_window = 1
        on = m(x, **kw).clone()
        again = m(x, **kw).clone()
        ad.attention_window = None
        off = m(x, **kw).clone()
    assert torch.equal(full, want)
    assert torch.equal(off, want)
    assert not torch.equal(on, want)
    assert torch.equal(on, again)


@pytest.mark.parametrize("fp8", [False, True])
def test_graphed_step_and_cross_kv_cache_bit_identical(fp8):
    from scail_b200 import sampler
    m = small_model(15, attention_window=1, fp8_attention=fp8, fp8_linear=fp8)
    g = torch.Generator().manual_seed(2)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    t, h, w = 5, 32, 32
    x0 = torch.randn(1, t, 16, h, w, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, h, w), concat_smpl_render=r(1, t, 16, h // 2, w // 2),
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
        m.mixins["adaln_layer"].attention_window = None
        dense = sampler.sample(m, x0.clone(), cond, uc, num_steps=2)
    torch.cuda.synchronize()
    assert torch.equal(xe, xg)
    assert torch.equal(plain, cached)
    assert not torch.equal(plain, dense)


def test_context_parallel_refused():
    class StubCP:
        size, rank = 2, 0

    m = small_model(1, attention_window=2)
    m.mixins["adaln_layer"].cp = StubCP()
    x, kw = small_inputs(2)
    with pytest.raises(NotImplementedError, match="attention_window"), torch.no_grad():
        m(x, **kw)


# ---------------------------------------------------------------- 5. the ABI refuses bad arguments
def test_abi_refuses_bad_counts_and_pointers():
    from scail_b200 import _lib
    h = _lib.lib()
    B, H, L, Lp = 1, 2, 300, 384  # 3 tiles
    d = H * 128
    ptr = torch.tensor([0, 3, 6, 9], device="cuda", dtype=torch.int32)
    idx = torch.tensor([0, 1, 2] * 3 + [0], device="cuda", dtype=torch.int32)
    x = torch.zeros(B * L, d, device="cuda", dtype=torch.bfloat16)
    out = torch.empty_like(x)
    P = lambda t: t.data_ptr()

    def att(**kw):
        a = dict(Q=P(x), ldq=d, K=P(x), ldk=d, V=P(x), ldv=d, out=P(out), ldo=d, B=B, H=H, q_len=L, kv_len=L, qb=L, kvb=L,
                 qt=B * L, kvt=B * L, scale=0.088, acc=0, ptr=P(ptr), idx=P(idx), nnz=9)
        a.update(kw)
        return h.scail_attention_sparse(*a.values(), None), h.scail_last_error()

    rc, err = att()
    assert rc == 0, err
    torch.cuda.synchronize()
    for kw, msg in [(dict(nnz=2), b"nnz"), (dict(nnz=10), b"nnz"), (dict(ptr=None), b"null tile map"),
                    (dict(idx=None), b"null tile map"), (dict(idx=P(idx) + 2), b"4-byte aligned"),
                    (dict(kv_len=299), b"self-attention only"), (dict(Q=None), b"null operand")]:
        rc, err = att(**kw)
        assert rc == -1 and msg in err, (kw, err)
    q8 = torch.zeros(B * L, d, device="cuda", dtype=torch.uint8)
    sc = torch.ones(B, H, Lp, device="cuda")
    vt = torch.zeros(B, H, 128, Lp, device="cuda", dtype=torch.uint8)
    vs = torch.ones(B, H, 128, device="cuda")

    def att8(**kw):
        a = dict(Q=P(q8), ldq=d, qs=P(sc), K=P(q8), ldk=d, ks=P(sc), vt=P(vt), vs=P(vs), out=P(out), ldo=d, B=B, H=H, hd=128,
                 L=L, Lp=Lp, scale=0.088, ptr=P(ptr), idx=P(idx), nnz=9)
        a.update(kw)
        return h.scail_attention_fp8_sparse(*a.values(), None), h.scail_last_error()

    rc, err = att8()
    assert rc == 0, err
    torch.cuda.synchronize()
    for kw, msg in [(dict(nnz=0), b"nnz"), (dict(nnz=10), b"nnz"), (dict(ptr=None), b"null tile map"),
                    (dict(ptr=P(ptr) + 1), b"4-byte aligned"), (dict(hd=64), b"head_dim"), (dict(L=400), b"L <= L_pad")]:
        rc, err = att8(**kw)
        assert rc == -1 and msg in err, (kw, err)
