"""The bf16 attention kernel's warpgroup ping-pong at the shapes that stress it: one, two, three and an odd number of key
tiles; a last CTA whose second consumer warpgroup has no valid query rows; a second key range that starts after a first
range ending mid-tile; an accumulating pass over 257 keys; and repeat launches on the same inputs.  Outputs are compared
with the fp32 oracle at the rel-L2 bound of tests/test_kernels_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def rnd(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(torch.bfloat16).cuda()


def oracle(q, k, v, B, H, nq, nkv):
    from oracle import dit_oracle as O
    D = H * 128
    return O.merge_heads(O.sdpa(O.heads(q.float().view(B, nq, D), H), O.heads(k.float().view(B, nkv, D), H),
                                O.heads(v.float().view(B, nkv, D), H)))


@pytest.mark.parametrize("B,H,nq,nkv", [(2, 2, 256, 100), (2, 2, 256, 256), (1, 3, 384, 300), (2, 2, 256, 833),
                                        (2, 2, 130, 300), (2, 1, 129, 257), (1, 2, 130, 1), (3, 1, 129, 640)])
def test_attention_tile_counts_and_ragged_rows(B, H, nq, nkv):
    from scail_b200 import ops
    D = H * 128
    q, k, v = rnd(B * nq, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    out = torch.zeros(B * nq, D, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, out, B, H, nq, nkv)
    torch.cuda.synchronize()
    r = rel(out.view(B, nq, D), oracle(q, k, v, B, H, nq, nkv))
    assert r < 6e-3, r


@pytest.mark.parametrize("ranges", [[(0, 200), (300, 150)], [(0, 64), (128, 40)], [(70, 130), (400, 257)]])
def test_attention_partial_second_range_after_ragged_first(ranges):
    """The first key range ends mid-tile, so the second range's tiles follow a masked tile; q_len = 130 leaves the last
    CTA's second warpgroup without valid rows."""
    from oracle import dit_oracle as O
    from scail_b200 import ops
    B, H, nq, nkv = 2, 2, 130, 700
    D = H * 128
    q, k, v = rnd(B * nq, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    o32 = torch.empty(B * nq, D, device="cuda", dtype=torch.float32)
    st = torch.empty(B * nq, H, 2, device="cuda", dtype=torch.float32)
    ops.attention_partial(q, k, v, o32, st, B, H, nq, ranges, kv_batch_rows=nkv)
    torch.cuda.synchronize()
    idx = torch.cat([torch.arange(o, o + n) for o, n in ranges]).cuda()
    ks, vs = k.view(B, nkv, D)[:, idx], v.view(B, nkv, D)[:, idx]
    n = idx.numel()
    ref = O.merge_heads(O.sdpa(O.heads(q.float().view(B, nq, D), H), O.heads(ks.float(), H), O.heads(vs.float(), H)))
    r = rel(o32.view(B, nq, D), ref)
    assert r < 6e-3, (r, n)


def test_attention_accumulate_257_keys():
    from scail_b200 import ops
    B, H, nq, nkv = 2, 2, 130, 257
    D = H * 128
    q, k, v = rnd(B * nq, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    base = rnd(B * nq, D, seed=4)
    out = base.clone()
    ops.attention(q, k, v, out, B, H, nq, nkv, accumulate=True)
    torch.cuda.synchronize()
    ref = base.float().view(B, nq, D) + oracle(q, k, v, B, H, nq, nkv)
    r = rel(out.view(B, nq, D), ref)
    assert r < 6e-3, r


def test_attention_repeat_launches_are_bit_identical():
    from scail_b200 import ops
    B, H, nq, nkv = 2, 4, 1000, 1500
    D = H * 128
    q, k, v = rnd(B * nq, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    a = torch.empty(B * nq, D, device="cuda", dtype=torch.bfloat16)
    b = torch.empty_like(a)
    ops.attention(q, k, v, a, B, H, nq, nkv)
    ops.attention(q, k, v, b, B, H, nq, nkv)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
