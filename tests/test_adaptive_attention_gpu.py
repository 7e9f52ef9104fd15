"""Content-adaptive block-sparse self-attention on the GPU: tile pooling against float64, the device selection against its
float64 restatement (tests/adaptive_oracle.py) on the kernel's own pooled tiles, the per-(batch, head) sparse kernels
against the fp32 masked softmax per head, bit-identity at mass 1, planted structure, the model against the fp32 oracle
masked with the maps the product chose, composition with the other opt-in modes, and ABI refusals.  TF32 is off."""
import math

import numpy as np
import pytest
import torch

from adaptive_oracle import csr_to_dense, expand_rows, masked_sdpa_bh, select_reference
from kernel_check import assert_close_bf16
from test_fp8_gpu import deq, quant_ref, rel, rnd
from test_sparse_attention_gpu import fp8_operands, heads, oracle, small_inputs, small_model

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn
LD = 15360  # the fused QKV buffer's row stride at 14B width


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def pool_ref(x64, B, H, L):
    """float64 tile means of x64 [B*L, H*128] -> [B, H, n, 128]."""
    n = -(-L // 128)
    xp = torch.zeros(B, n * 128, H, 128, dtype=torch.float64, device=x64.device)
    xp[:, :L] = x64.view(B, L, H, 128)
    cnt = torch.clamp(L - 128 * torch.arange(n, device=x64.device), max=128).double()
    return (xp.view(B, n, 128, H, 128).sum(2) / cnt[None, :, None, None]).permute(0, 2, 1, 3)


def bh_dense(ptr, idx):
    """Device per-(b, h) maps -> bool [B, H, n, n] (torch, CPU) after checking every map with ops.check_tile_map."""
    from scail_b200 import ops, sparse
    B, H, n1 = ptr.shape
    n = n1 - 1
    out = torch.zeros(B, H, n, n, dtype=torch.bool)
    for (b, h), (p, i) in sparse.bh_maps_host(ptr, idx).items():
        ops.check_tile_map(p, i, n * 128, n * 128)
        out[b, h] = torch.from_numpy(csr_to_dense(p, i, n))
    return out


def upload_maps(tm):
    """bool [B, H, n, n] -> device (ptr int32 [B, H, n + 1], idx int32 [B, H, n * n])."""
    B, H, n, _ = tm.shape
    ptr = torch.zeros(B, H, n + 1, dtype=torch.int32)
    idx = torch.zeros(B, H, n * n, dtype=torch.int32)
    for b in range(B):
        for h in range(H):
            r, c = np.nonzero(tm[b, h].numpy())
            ptr[b, h, 1:] = torch.from_numpy(np.cumsum(tm[b, h].sum(1).numpy()))
            idx[b, h, :c.size] = torch.from_numpy(c.astype(np.int32))
    return ptr.cuda(), idx.cuda()


def wide_slabs(B, L, H, seed):
    """bf16 Q and K slabs [B*L, H*128] as views of one buffer with row stride 15 360."""
    d = H * 128
    buf = rnd(B * L, LD, seed=seed)
    return buf[:, :d], buf[:, 5120:5120 + d]


# ---------------------------------------------------------------- 1. pooling
@pytest.mark.parametrize("L", [129, 130, 1000, 27904])
def test_tile_pool_against_float64(L):
    from scail_b200 import ops
    B, H = (1, 40) if L == 27904 else (2, 3)
    q, k = wide_slabs(B, L, H, L)
    assert q.stride(0) == LD
    for x in (q, k):
        got = ops.tile_pool(x, B, H, L)
        again = ops.tile_pool(x, B, H, L)
        want = pool_ref(x.double(), B, H, L)
        torch.cuda.synchronize()
        assert torch.equal(got, again)
        assert ((got.double() - want).abs() <= 1e-6 * want.abs() + 1e-30).all()
    # e4m3 codes in a 15 360-wide buffer, times their per-(token, head) scales
    d = H * 128
    q8, qs = quant_ref(q.reshape(-1, 128))
    codes = torch.zeros(B * L, LD, dtype=torch.uint8, device="cuda")
    codes[:, 128:128 + d] = q8.view(torch.uint8).view(B * L, d)
    x8 = codes[:, 128:128 + d].view(FP8)
    Lp = -(-L // 128) * 128
    scale = torch.zeros(B, H, Lp, device="cuda")
    scale[:, :, :L] = (qs * 1.37).view(B, L, H).permute(0, 2, 1)
    got = ops.tile_pool(x8, B, H, L, x_scale=scale)
    again = ops.tile_pool(x8, B, H, L, x_scale=scale)
    x64 = (x8.float().double().view(B, L, H, 128) * scale[:, :, :L].permute(0, 2, 1).double()[..., None]).view(B * L, d)
    want = pool_ref(x64, B, H, L)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert ((got.double() - want).abs() <= 1e-6 * want.abs() + 1e-30).all()


# ---------------------------------------------------------------- 2. selection
def structured(B, L, H, seed, amp=3.0):
    """Q, K slabs whose tiles carry a shared component (amplitude amp) plus token noise: the tile scores spread over several
    units (sharply peaked rows, as in attention with structure) rather than the near-uniform scores of i.i.d. tokens, so
    few rows sit within rounding of their cutoff."""
    d = H * 128
    n = -(-L // 128)
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for _ in range(2):
        base = (torch.randn(B, n, 1, d, generator=g) * amp).expand(B, n, 128, d).reshape(B, n * 128, d)[:, :L]
        out.append((base + torch.randn(B, L, d, generator=g)).reshape(B * L, d).to(torch.bfloat16).cuda())
    return out


@pytest.mark.parametrize("L,n_ref,mass,cap", [(1000, 130, 0.9, None), (1000, 0, 0.5, 2), (27904, 1024, 0.9, None),
                                              (27904, 1024, 0.95, 40), (27904, 1024, 0.0, None), (27904, 1560, 1.0, 5)])
def test_selection_against_float64_restatement(L, n_ref, mass, cap):
    from scail_b200 import ops, sparse
    B, H = (2, 3) if L < 5000 else (1, 16)
    q, k = structured(B, L, H, seed=L + int(100 * mass))
    n = -(-L // 128)
    ws = {}
    buf = lambda name, shape, dtype: ws.setdefault(name, torch.empty(shape, device="cuda", dtype=dtype))
    ptr, idx = sparse.AdaptiveTiles(mass, cap).select(q, k, B, H, L, n_ref, buf)
    got_t = bh_dense(ptr, idx)
    got, ptr1 = got_t.numpy(), ptr.clone()
    want, near = select_reference(ws["ada_qbar"].cpu().numpy(), ws["ada_kbar"].cpu().numpy(), L, n_ref, mass, cap, band=1e-5)
    n_ref_t = -(-n_ref // 128)
    assert got[..., :n_ref_t].all() and got[..., np.arange(n), np.arange(n)].all()  # forced tiles
    diff = (got != want).any(-1)
    assert not (diff & ~near).any(), np.argwhere(diff & ~near)[:5]
    assert near.mean() <= 1e-3, near.mean()
    ptr2, idx2 = sparse.AdaptiveTiles(mass, cap).select(q, k, B, H, L, n_ref, buf)  # a repeat launch: the same maps
    assert torch.equal(ptr2, ptr1) and torch.equal(bh_dense(ptr2, idx2), got_t)
    print(f"L={L} mass={mass} cap={cap}: density {got.mean():.3f}, rows at the cutoff {near.sum()} of {near.size}")


# ---------------------------------------------------------------- 3. the per-(b, h) kernels
def planted(B, H, L, plant, seed, c=11.7, noise=0.5):
    """Q, K, V bf16 [B*L, H*128]: K tile k of head h carries c along channel k % 128 of that head; query tile q of (b, h)
    carries c along the channels of the tiles plant[b][h][q].  Then the planted tiles hold nearly the whole softmax row."""
    d = H * 128
    n = -(-L // 128)
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randn(B, L, H, 128, generator=g) * noise
    k = torch.randn(B, L, H, 128, generator=g) * noise
    v = torch.randn(B, L, H, 128, generator=g)
    for t in range(n):
        k[:, 128 * t:128 * t + 128, :, t % 128] += c
    for b in range(B):
        for h in range(H):
            for t in range(n):
                for p in plant[b][h][t]:
                    q[b, 128 * t:128 * t + 128, h, p % 128] += c
    return [x.reshape(B * L, d).to(torch.bfloat16).cuda() for x in (q, k, v)]


def masked_chain_fp8_bh(q, k, v, tm, chunk=256):
    """The restated fp8 chain (test_sparse_attention_gpu.masked_chain_fp8) under per-(b, h) tile masks."""
    B, H, L, D = q.shape
    qd = deq(*quant_ref(q.reshape(-1, D))).view(B, H, L, D)
    kd = deq(*quant_ref(k.reshape(-1, D))).view(B, H, L, D)
    vd = deq(*quant_ref(v.transpose(-1, -2).reshape(-1, L))).view(B, H, D, L).transpose(-1, -2)
    out = torch.empty(B, H, L, D, device=q.device)
    kt = kd.transpose(-1, -2)
    for i in range(0, L, chunk):
        j = min(L, i + chunk)
        s = ((qd[:, :, i:j] @ kt) * D ** -0.5).masked_fill_(~expand_rows(tm, i, j, L), float("-inf"))
        p = torch.exp(s - s.amax(-1, keepdim=True)) * 256.0
        out[:, :, i:j] = (p.to(FP8).float() @ vd) / p.sum(-1, keepdim=True)
        del s, p
    return out


@pytest.mark.parametrize("B,H,L", [(2, 3, 1000), (1, 2, 27904)])
def test_per_head_kernels_against_masked_softmax_per_head(B, H, L):
    from scail_b200 import ops
    n = -(-L // 128)
    rng = np.random.default_rng(L)
    tm = torch.from_numpy(rng.random((B, H, n, n)) < (0.3 if n < 20 else 0.05))
    plant = [[[[int(rng.integers(n))] for _ in range(n)] for _ in range(H)] for _ in range(B)]
    for b in range(B):
        for h in range(H):
            for t in range(n):
                tm[b, h, t, t] = True
                tm[b, h, t, plant[b][h][t][0]] = True
    assert not torch.equal(tm[0, 0], tm[0, 1])
    q, k, v = planted(B, H, L, plant, seed=L)
    d = H * 128
    ptr, idx = upload_maps(tm)
    tmc = tm.cuda()
    out = torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16)
    ops.attention_sparse_bh(q, k, v, out, B, H, L, ptr, idx)
    want = masked_sdpa_bh(heads(q, B, L, H), heads(k, B, L, H), heads(v, B, L, H), tmc).transpose(1, 2).reshape(B * L, d)
    torch.cuda.synchronize()
    c = assert_close_bf16(out, want, f"bf16 per-(b, h), L={L}", elem_rel=2.0 ** -7, elem_abs=2.0 ** -8)
    print(f"bf16 per-(b, h) L={L}: rel-L2 {c.rel_l2:.3e}, worst |d|/bound {c.worst_ratio:.3f}")
    # a kernel that read another head's row would miss the planted tile: whole rows would move
    shared = torch.empty_like(out)
    ops.attention_sparse_bh(q, k, v, shared, B, H, L, ptr[:1, :1].expand(B, H, -1).contiguous(),
                            idx[:1, :1].expand(B, H, -1).contiguous())
    assert rel(shared, want) > 0.1
    q8, qs, k8, ks, vt, vs = fp8_operands(torch.cat([q, k, v], 1), B, H, L)
    ops.attention_fp8_sparse_bh(q8, qs, k8, ks, vt, vs, out, B, H, L, ptr, idx)
    chain = masked_chain_fp8_bh(heads(q, B, L, H), heads(k, B, L, H), heads(v, B, L, H), tmc).transpose(1, 2).reshape(B * L, d)
    torch.cuda.synchronize()
    e, e_chain = rel(out, want), rel(chain, want)
    print(f"fp8 per-(b, h) L={L}: ours vs fp32 {e:.3e} | restated masked fp8 chain vs fp32 {e_chain:.3e}")
    assert torch.isfinite(out.float()).all() and e <= 1.25 * e_chain + 1e-3, (e, e_chain)


# ---------------------------------------------------------------- 4. mass 1 is the dense kernel, bit for bit
@pytest.mark.parametrize("B,H,L", [(2, 2, 129), (2, 2, 130), (2, 3, 1000), (1, 8, 27904)])
def test_mass_one_is_bit_identical_to_the_dense_kernels(B, H, L):
    from scail_b200 import ops, sparse
    d = H * 128
    qkv = rnd(B * L, 3 * d, seed=L)
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    buf = lambda name, shape, dtype: torch.empty(shape, device="cuda", dtype=dtype)
    a, b = (torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    ptr, idx = sparse.AdaptiveTiles(1.0).select(q, k, B, H, L, 0, buf)
    assert bh_dense(ptr, idx).all()
    ops.attention(q, k, v, a, B, H, L, L)
    ops.attention_sparse_bh(q, k, v, b, B, H, L, ptr, idx)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    q8, qs, k8, ks, vt, vs = fp8_operands(qkv, B, H, L)
    ptr, idx = sparse.AdaptiveTiles(1.0).select(q8, k8, B, H, L, 0, buf, q_scale=qs, k_scale=ks)
    ops.attention_fp8(q8, qs, k8, ks, vt, vs, a, B, H, L)
    ops.attention_fp8_sparse_bh(q8, qs, k8, ks, vt, vs, b, B, H, L, ptr, idx)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


@pytest.mark.parametrize("fp8_attention", [False, True])
def test_mass_one_and_toggling_off_reproduce_the_dense_forward(fp8_attention):
    from scail_b200 import sparse
    x, kw = small_inputs(5)
    m = small_model(6, fp8_attention=fp8_attention)
    ad = m.mixins["adaln_layer"]
    with torch.no_grad():
        want = m(x, **kw).clone()
        ad.attention_adaptive = sparse.AdaptiveTiles(1.0)
        full = m(x, **kw).clone()
        ad.attention_adaptive = sparse.AdaptiveTiles(0.9, max_tiles=2)
        on = m(x, **kw).clone()
        again = m(x, **kw).clone()
        ad.attention_adaptive = None
        off = m(x, **kw).clone()
    assert torch.equal(full, want) and torch.equal(off, want)
    assert not torch.equal(on, want) and torch.equal(on, again)


# ---------------------------------------------------------------- 5. planted structure
def test_planted_structure_is_found_exactly():
    from scail_b200 import ops, sparse
    B, H, L, n_ref = 2, 3, 2000, 130  # 16 tiles, the last holding 80 keys; ref tiles 0 and 1
    n = -(-L // 128)
    rng = np.random.default_rng(9)
    plant = [[[sorted(rng.choice([j for j in range(2, n) if j != t], 2, replace=False).tolist()) for t in range(n)]
              for _ in range(H)] for _ in range(B)]
    q, k, v = planted(B, H, L, plant, seed=4)
    d = H * 128
    buf = lambda name, shape, dtype: torch.empty(shape, device="cuda", dtype=dtype)
    ptr, idx = sparse.AdaptiveTiles(0.9).select(q, k, B, H, L, n_ref, buf)
    got = bh_dense(ptr, idx)
    for b in range(B):
        for h in range(H):
            for t in range(n):
                want = sorted({0, 1, t} | set(plant[b][h][t]))
                assert torch.nonzero(got[b, h, t]).flatten().tolist() == want, (b, h, t)
    out, dense = (torch.empty(B * L, d, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    ops.attention_sparse_bh(q, k, v, out, B, H, L, ptr, idx)
    ops.attention(q, k, v, dense, B, H, L, L)
    torch.cuda.synchronize()
    e = rel(out, dense)
    print(f"planted structure: density {got.float().mean():.3f}, rel-L2 against dense {e:.3e}")
    assert e <= 1e-2


# ---------------------------------------------------------------- 6. the model against the masked fp32 oracle
def masked_oracle(args, maps):
    """oracle() (test_sparse_attention_gpu) with each layer's self-attention masked per (b, h) by the maps recorded during
    our forward, in layer order."""
    import oracle.dit_oracle as O
    old = O.sdpa
    layers = iter(maps)

    def sdpa(q, k, v):
        if q.dtype != torch.float32 or q.shape[-2] != k.shape[-2]:
            return old(q, k, v)
        return masked_sdpa_bh(q, k, v, bh_dense(*next(layers)).cuda())

    O.sdpa = sdpa
    try:
        with torch.no_grad(), torch.device("cuda"):
            return O.dit_forward(*args)
    finally:
        O.sdpa = old


def check_model(what, m, x, kw, args, adaptive):
    from scail_b200 import sparse
    ad = m.mixins["adaln_layer"]
    with torch.no_grad():
        dense = m(x, **kw).float()
        ad.attention_adaptive = adaptive
        sparse.RECORD = []
        try:
            got = m(x, **kw).float()
            maps = sparse.RECORD
        finally:
            sparse.RECORD = None
            ad.attention_adaptive = None
    assert len(maps) == m.num_layers
    density = float(np.mean([bh_dense(*mp).float().mean() for mp in maps]))
    assert density < 0.9
    want, want_dense = masked_oracle(args, maps), oracle(args)
    e, e_dense = rel(got, want), rel(dense, want_dense)
    print(f"{what}, {adaptive} (density {density:.3f}): ours vs masked oracle {e:.3e} | dense vs oracle {e_dense:.3e}")
    assert e <= 1.25 * e_dense + 1e-3, (e, e_dense)


def test_small_model_against_masked_oracle():
    from scail_b200 import sparse
    m = small_model(3)
    x, kw = small_inputs(4)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    args = (sd, x.float(), kw["timesteps"], kw["context"].float(), kw["ref_concat"].float(),
            kw["concat_smpl_render"].float(), kw["image_clip_features"].float(), 2, 2)
    check_model("small 2-layer model", m, x, kw, args, sparse.AdaptiveTiles(0.9, max_tiles=3))


def test_full_width_block_at_config_A_against_masked_oracle():
    """One 14B-width block (5120 / 40 heads / 13824) at N = 27 904, b = 1."""
    from scail_b200 import sparse
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
    check_model("config-A block (N=27904, b=1)", m, x, kw, args, sparse.AdaptiveTiles(0.9, max_tiles=40))


# ---------------------------------------------------------------- 7. composition
def sampler_inputs(seed=2, t=5, h=32, w=32):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    x0 = torch.randn(1, t, 16, h, w, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, h, w), concat_smpl_render=r(1, t, 16, h // 2, w // 2),
                image_clip_features=r(1, 257, 1280))
    return x0, cond, dict(crossattn=r(1, 24, 64))


@pytest.mark.parametrize("fp8", [False, True])
def test_graphed_step_and_cross_kv_cache_bit_identical(fp8):
    from scail_b200 import sampler, sparse
    m = small_model(15, attention_adaptive=sparse.AdaptiveTiles(0.9, max_tiles=2), fp8_attention=fp8, fp8_linear=fp8)
    x0, cond, uc = sampler_inputs()
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
        m.mixins["adaln_layer"].attention_adaptive = None
        dense = sampler.sample(m, x0.clone(), cond, uc, num_steps=2)
    torch.cuda.synchronize()
    assert torch.equal(xe, xg)
    assert torch.equal(plain, cached)
    assert not torch.equal(plain, dense)


def test_graphed_step_with_fp8_and_step_cache_bit_identical():
    from scail_b200 import sampler, sparse
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(16, attention_adaptive=sparse.AdaptiveTiles(0.8, max_tiles=3), fp8_attention=True, fp8_linear=True)
    x0, cond, uc = sampler_inputs(3)
    sig = sampler.make_flow_timesteps(50, 5.0)
    ce, cg = FirstBlockCache(0.0), FirstBlockCache(0.0)
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, step_cache=cg)
        for i, thr in enumerate([0.0, math.inf, 0.0, math.inf]):
            ce.threshold = cg.threshold = thr
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=ce)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(xe, xg), f"step {i}"


def test_context_parallel_refused():
    from scail_b200 import sparse

    class StubCP:
        size, rank = 2, 0

    m = small_model(1, attention_adaptive=sparse.AdaptiveTiles(0.9))
    m.mixins["adaln_layer"].cp = StubCP()
    x, kw = small_inputs(2)
    with pytest.raises(NotImplementedError, match="attention_adaptive"), torch.no_grad():
        m(x, **kw)


# ---------------------------------------------------------------- 8. the ABI refuses bad arguments
def test_abi_refuses_null_misaligned_and_inconsistent_arguments():
    from scail_b200 import _lib
    h = _lib.lib()
    B, H, L, Lp, n = 1, 2, 300, 384, 3
    d = H * 128
    P = lambda t: t.data_ptr()
    x = torch.zeros(B * L, d, device="cuda", dtype=torch.bfloat16)
    out = torch.empty_like(x)
    ptr = torch.zeros(B, H, n + 1, device="cuda", dtype=torch.int32)
    idx = torch.zeros(B, H, n * n, device="cuda", dtype=torch.int32)
    qbar = torch.zeros(B, H, n, 128, device="cuda")
    scratch = torch.zeros(B * H * n * 2, device="cuda", dtype=torch.int32)
    sc = torch.ones(B, H, Lp, device="cuda")

    def call(fn, base, kw):
        a = dict(base)
        a.update(kw)
        return getattr(h, fn)(*a.values(), None), h.scail_last_error()

    sel = dict(qbar=P(qbar), kbar=P(qbar), B=B, H=H, L=L, n_ref=0, mass=1.0, cap=-1, ptr=P(ptr), ps=n + 1, idx=P(idx),
               ids=n * n, scratch=P(scratch), slen=scratch.numel())
    rc, err = call("scail_attention_select_tiles", sel, {})
    assert rc == 0, err
    att = dict(Q=P(x), ldq=d, K=P(x), ldk=d, V=P(x), ldv=d, out=P(out), ldo=d, B=B, H=H, L=L, qb=L, kvb=L, qt=B * L,
               kvt=B * L, scale=0.088, ptr=P(ptr), ps=n + 1, idx=P(idx), ids=n * n)
    rc, err = call("scail_attention_sparse_bh", att, {})
    assert rc == 0, err
    q8 = torch.zeros(B * L, d, device="cuda", dtype=torch.uint8)
    vt = torch.zeros(B, H, 128, Lp, device="cuda", dtype=torch.uint8)
    att8 = dict(Q=P(q8), ldq=d, qs=P(sc), K=P(q8), ldk=d, ks=P(sc), vt=P(vt), vs=P(sc), out=P(out), ldo=d, B=B, H=H, hd=128,
                L=L, Lp=Lp, scale=0.088, ptr=P(ptr), ps=n + 1, idx=P(idx), ids=n * n)
    rc, err = call("scail_attention_fp8_sparse_bh", att8, {})
    assert rc == 0, err
    pool = dict(x=P(x), ldx=d, xs=None, fp8=0, out=P(qbar), B=B, H=H, L=L, Lp=0)
    rc, err = call("scail_attention_tile_pool", pool, {})
    assert rc == 0, err
    torch.cuda.synchronize()
    cases = {
        "scail_attention_select_tiles": (sel, [
            (dict(qbar=None), b"null operand"), (dict(scratch=None), b"null operand"), (dict(ptr=None), b"null tile map"),
            (dict(qbar=P(qbar) + 4), b"16-byte aligned"), (dict(idx=P(idx) + 2), b"4-byte aligned"),
            (dict(ps=n), b"ptr_stride"), (dict(ids=n * n - 1), b"idx_stride"), (dict(slen=11), b"scratch holds"),
            (dict(mass=math.nan), b"mass"), (dict(mass=1.5), b"mass"), (dict(cap=-2), b"max_tiles"),
            (dict(n_ref=301), b"n_ref"), (dict(L=0), b"L=0")]),
        "scail_attention_sparse_bh": (att, [
            (dict(ptr=None), b"null tile map"), (dict(idx=P(idx) + 1), b"4-byte aligned"), (dict(ps=0), b"ptr_stride"),
            (dict(ids=n), b"idx_stride"), (dict(Q=None), b"null operand")]),
        "scail_attention_fp8_sparse_bh": (att8, [
            (dict(idx=None), b"null tile map"), (dict(ps=n), b"ptr_stride"), (dict(ids=0), b"idx_stride"),
            (dict(hd=64), b"head_dim"), (dict(L=400, ps=5, ids=16), b"L <= L_pad")]),
        "scail_attention_tile_pool": (pool, [
            (dict(x=None), b"null operand"), (dict(out=None), b"null operand"), (dict(fp8=2), b"fp8=2"),
            (dict(fp8=1), b"x_scale"), (dict(xs=P(sc)), b"x_scale"), (dict(ldx=d - 8), b"ldx"),
            (dict(out=P(qbar) + 2), b"4-byte aligned"), (dict(fp8=1, xs=P(sc), Lp=300), b"L_pad")]),
    }
    for fn, (base, bad) in cases.items():
        for kw, msg in bad:
            rc, err = call(fn, base, kw)
            assert rc == -1 and msg in err, (fn, kw, err)
