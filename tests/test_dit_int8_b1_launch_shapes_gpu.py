"""The INT8 Q·Kᵀ and conditional-only (b = 1) DiT launches of the 14B step against fp32, element by element.

test_every_int8_b1_launch_matches_fp32: the full-width two-block random model of test_dit_launch_shapes_gpu.py runs, at
21x64x64 (N = 27 904), 21x60x104 (N = 42 510, 14 keys in the last tile) and 21x64x112 (N = 48 832, 64 keys in the last
tile):
  - one sampler.sampler_step (CFG batch b = 2) in each INT8 mode: fp8_attention="int8_qk" dense, with the window-2 map,
    with AdaptiveTiles(0.9, max_tiles=40), and dense with fp8 linears;
  - the conditional row alone (b = 1: a skipped step of CFGCache, a rank of the 2-GPU CFG split or of HybridParallel) in
    every mode: the six of test_dit_launch_shapes_gpu.MODES and the four INT8 ones, called as the CFG cache calls it (the
    fp32 latent, one timestep, the cond row of prepare_context);
  - CFGCache(inf) over three sampler steps, in bf16 and in int8_qk: steps 0 and 1 are full and step 2 conditional-only.
    test_cfg_cache_skip_launches_are_the_direct_b1_ones asserts that step 2 makes no launch the direct b = 1 forwards did
    not, so those forwards stand for what the cache launches.
Every DiT entry point and the three INT8 ones are recorded by kernel_check.recording, and each distinct launch is re-run on
fresh seeded data inside sentinel buffers (test_dit_launch_shapes_gpu.Slab: 128 trailing sentinel rows).  The INT8 entry
points are checked here:
  rmsnorm_rope_int8q: codes and scales bit for bit test_int8qk_attention_gpu.heads_ref of rmsnorm_rope's output on the
    geometry's real RoPE tables, the scales zero in [L, L_pad) (attention_int8qk reads that padding), the K slab normalised
    in bf16 bit for bit as rmsnorm_rope writes it, the Q slab and every other column untouched;
  quant_k_int8: k-bar within one fp32 ulp of the fp64 mean over the L valid keys (a ragged mean at 42 510 and 48 832, on
    keys with a per-(batch, channel) offset), codes and scales of K' = K - k-bar bit for bit;
  attention_int8qk, dense, window and per-(batch, head): the planted-key data of test_dit_launch_shapes_gpu._attention_data
    (_adaptive_data for per-(batch, head) maps) against the fp32 softmax and the restated int8 chain, to the fp8 rule
    (_fp8_verdict: rel-L2 <= 1.25x the chain's, the worst (batch, head, 128-query) block <= 2x the chain's worst, every
    planted row), and bit-identical to a launch on compact operands.  The K scales in [L, L_pad) hold each (batch, head)'s
    mean scale instead of the zeros the quantisers write: the kernel must mask those keys, not lean on a zero scale, and a
    key leaked past L then carries a real logit.
Every other launch, b = 1 included, goes through test_dit_launch_shapes_gpu.CHECKS (tile_pool with its INT8 form).

test_full_width_block_at_480x832_int8_vs_oracle: one full-width block at 21x60x104, b = 2, in int8_qk with bf16 linears,
against oracle/dit_oracle.py in fp32, next to the same block with fp8 attention."""
import math
import time

import pytest
import torch

from kernel_check import recording
from test_dit_launch_shapes_gpu import (ADAPTIVE, BF, CHECKS, GEOMETRIES, MODES, OPS, Slab, _adaptive_data, _attention_data,
                                        _attention_ref, _describe, _exact, _fields, _flat, _fp8_verdict, _no_tf32, _rand,
                                        _rope_geometry, _tile_key, _tile_matrix, _view, full_width_model, rel, step_inputs)
from test_adaptive_attention_gpu import upload_maps
from test_fp8_attention_gpu import pad, vt_ref
from test_int8qk_attention_gpu import heads_ref, kbar_fp64, ulp_f32
from test_scale_gpu import sdpa_fp32_chunked

pytestmark = pytest.mark.gpu
_no_tf32 = _no_tf32  # autouse: TF32 off in every test of this module

INT8_OPS = ("rmsnorm_rope_int8q", "quant_k_int8", "attention_int8qk")
ALL_OPS = OPS + INT8_OPS
INT8_MODES = {"int8": dict(fp8_attention="int8_qk"), "int8, window 2": dict(fp8_attention="int8_qk", attention_window=2),
              "int8, adaptive": dict(fp8_attention="int8_qk", attention_adaptive=True),
              "int8, fp8 linears": dict(fp8_attention="int8_qk", fp8_linear=True)}
B1_MODES = {**MODES, **INT8_MODES}
CACHE_MODES = ("bf16", "int8")


# ---------------------------------------------------------------- recording
def _fields_int8(name, a):
    if name == "rmsnorm_rope_int8q":
        buf = a["buf"]
        return dict(rows=buf.shape[0], L=a["rows_per_batch"], D=a["D"], buf=_view(buf), width=buf.shape[1],
                    slabs=tuple(o for o, _ in a["slabs"]), q8=_view(a["q8"]), L_pad=a["q_scale"].shape[-1],
                    rope=_rope_geometry(a["cos"]), eps=float(a["eps"])), 1
    if name == "quant_k_int8":
        return dict(B=a["B"], H=a["H"], L=a["L"], k=_view(a["k"]), k8=_view(a["k8"]), L_pad=a["scale"].shape[-1]), 1
    if name == "attention_int8qk":
        bh = a["bh_maps"]
        return dict(B=a["B"], H=a["H"], L=a["L"], q=_view(a["q8"]), k=_view(a["k8"]), out=_view(a["out"]),
                    L_pad=a["q_scale"].shape[-1], scale=float(a["scale"] or 1.0 / math.sqrt(128)),
                    tiles=_tile_key(a["tiles"]), bh=None if bh is None else (bh[0].shape[2], bh[1].shape[2])), 1
    return _fields(name, a)


def _set_mode(ad, mode):
    from scail_b200 import sparse
    ad.fp8_linear = mode.get("fp8_linear", False)
    ad.fp8_attention = mode.get("fp8_attention", False)
    ad.attention_window = mode.get("attention_window")
    ad.attention_adaptive = sparse.AdaptiveTiles(*ADAPTIVE) if mode.get("attention_adaptive") else None


@pytest.fixture(scope="module")
def workload():
    """{"launches": [(op, key)] in first-call order, "b1": {geometry: set of keys of the direct b = 1 forwards},
    "skip": {(geometry, cache mode): set of keys of the conditional-only step}}."""
    from scail_b200 import dit, ops, sampler
    from scail_b200.cfg_cache import CFGCache
    m = full_width_model(2)
    ad = m.mixins["adaln_layer"]
    sig = sampler.make_flow_timesteps(50, 5.0)
    b1, skip = {}, {}
    with torch.no_grad(), recording(ops, ALL_OPS, _fields_int8) as seen:
        for i, (geo, (t, h, w)) in enumerate(GEOMETRIES.items()):
            x0, cond, uc = step_inputs(10 + i, t, h, w)
            for mode in INT8_MODES.values():
                _set_mode(ad, mode)
                sampler.sampler_step(m, x0.clone(), sig[0], sig[1], cond, uc, 4.0)
            # the conditional-only forward as CFGCache.cond_forward makes it: fp32 latent, one timestep, ctx[1:2]
            ctx = sampler.prepare_context(cond, uc)[1:2]
            ts = torch.full((1,), float(sig[2]) * 1000.0, device="cuda")
            with recording(ops, ALL_OPS, _fields_int8) as direct:
                for mode in B1_MODES.values():
                    _set_mode(ad, mode)
                    m(x0.clone(), timesteps=ts, context=ctx, y=None, ref_concat=cond["ref_concat"],
                      concat_smpl_render=cond["concat_smpl_render"], image_clip_features=cond["image_clip_features"],
                      concat_images=None)
            b1[geo] = set(direct)
            for cm in CACHE_MODES:
                _set_mode(ad, B1_MODES[cm])
                c, x = CFGCache(math.inf), x0.clone()
                for j in range(2):
                    sampler.sampler_step(m, x, sig[j], sig[j + 1], cond, uc, 4.0, cfg_cache=c)
                with recording(ops, ALL_OPS, _fields_int8) as cached:
                    sampler.sampler_step(m, x, sig[2], sig[3], cond, uc, 4.0, cfg_cache=c)
                assert [s for _, s in c.history] == [False, False, True], c.history
                skip[(geo, cm)] = set(cached)
                del c
            _set_mode(ad, {})
    torch.cuda.synchronize()
    del m, ad
    dit._WS.bufs.clear()
    torch.cuda.empty_cache()
    return dict(launches=[(name, dict(k)) for (name, k) in seen], b1=b1, skip=skip)


@pytest.fixture(scope="module")
def launches(workload):
    return workload["launches"]


# ---------------------------------------------------------------- the INT8 entry points vs their restatements
def _scales(B, H, Lp, fill=7.0):
    """A scale tensor [B, H, L_pad] full of `fill` with sentinels around it: (slab, view)."""
    return _flat(torch.full((B, H, Lp), fill, device="cuda"))


def check_rmsnorm_rope_int8q(ops, f, g):
    from scail_b200 import rope
    rows, L, D, eps, Lp = f["rows"], f["L"], f["D"], f["eps"], f["L_pad"]
    B, H = rows // L, D // 128
    assert len(f["slabs"]) == 2 and Lp == pad(L)
    data = _rand(g, rows, f["width"], scale=2.0)
    slabs = [(o, 1 + _rand(g, D, scale=0.1)) for o in f["slabs"]]
    cos = sin = None
    if f["rope"] is not None:  # the geometry's real tables, as check_rmsnorm_rope
        *geo, row = f["rope"]
        cos, sin = rope.build_tables("cuda", 128, *geo)
        cos, sin = cos[row:row + L], sin[row:row + L]
    buf = Slab(data, f["buf"])
    q8 = Slab(torch.zeros(rows, D, device="cuda", dtype=torch.int8), f["q8"])
    S, qs = _scales(B, H, Lp)
    ops.rmsnorm_rope_int8q(buf.v, L, D, slabs, q8.v, qs, cos, sin, eps=eps)
    torch.cuda.synchronize()
    for s in (buf, q8, S):
        s.check("rmsnorm_rope_int8q")
    ref = data.clone()
    ops.rmsnorm_rope(ref, L, D, slabs, cos, sin, eps=eps)  # pinned to fp32 by check_rmsnorm_rope at the same geometry
    (oq, _), (ok, _) = slabs
    qr, sr = heads_ref(ref[:, oq:oq + D], B, H, L)
    assert not qs[:, :, L:].any(), "rmsnorm_rope_int8q: Q scales in [L, L_pad) are not zero"
    _exact(qs, sr, "rmsnorm_rope_int8q scales")
    _exact(q8.v, qr, "rmsnorm_rope_int8q codes")
    _exact(buf.v[:, ok:ok + D], ref[:, ok:ok + D], "rmsnorm_rope_int8q: the K slab as rmsnorm_rope writes it")
    other = torch.ones(f["width"], dtype=torch.bool)
    other[ok:ok + D] = False
    _exact(buf.v[:, other.cuda()], data[:, other.cuda()], "rmsnorm_rope_int8q: the Q slab and the other columns")
    return f"exact; scales zero in [{L}, {Lp})", 0.0


def check_quant_k_int8(ops, f, g):
    B, H, L, Lp = f["B"], f["H"], f["L"], f["L_pad"]
    d = H * 128
    assert Lp == pad(L)
    off = torch.randn(B, 1, d, device="cuda", generator=g) * 2.0  # a per-(batch, channel) offset: the mean matters
    k = (torch.randn(B, L, d, device="cuda", generator=g) * 2.0 + off).to(BF).view(B * L, d)
    K = Slab(k, f["k"])
    K8 = Slab(torch.zeros(B * L, d, device="cuda", dtype=torch.int8), f["k8"])
    S, ks = _scales(B, H, Lp)
    M, kb = _flat(torch.full((B, d), 7.0, device="cuda"))
    P, part = _flat(torch.full((ops.quant_k_int8_partial_len(B, H, L) // d, d), 7.0, device="cuda", dtype=torch.float64))
    ops.quant_k_int8(K.v, B, H, L, K8.v, ks, kb, part.view(-1))
    torch.cuda.synchronize()
    for s in (K, K8, S, M, P):
        s.check("quant_k_int8")
    _exact(K.v, k, "quant_k_int8: its input")
    want = kbar_fp64(k, B, L)
    d_bar = (kb - want).abs()
    assert (d_bar <= ulp_f32(want)).all(), f"quant_k_int8: k-bar off the fp64 mean by up to {float(d_bar.max()):.3g}"
    kr, ksr = heads_ref((k.float().view(B, L, d) - kb[:, None, :]).view(B * L, d), B, H, L)
    _exact(ks, ksr, "quant_k_int8 scales")
    _exact(K8.v, kr, "quant_k_int8 codes")
    return f"exact; k-bar within one fp32 ulp of the fp64 mean over {L} keys (max |d| {float(d_bar.max()):.2g})", 0.0


def check_attention_int8qk(ops, f, g):
    from scail_b200 import sparse as S
    B, H, L, Lp = f["B"], f["H"], f["L"], f["L_pad"]
    d = H * 128
    assert Lp == pad(L)
    tm = tiles = None
    if f["bh"] is not None:
        q, k, v, tm, planted = _adaptive_data(ops, g, f)
        mask = tm.cuda()
    else:
        tiles = _tile_matrix(f["tiles"]) if f["tiles"] is not None else None
        q, k, v, planted = _attention_data(g, dict(B=B, H=H, q_len=L, kv_len=L, scale=f["scale"]), tiles)
        mask = tiles
    qi, qis = heads_ref(q, B, H, L)
    kbar = kbar_fp64(k, B, L)
    ki, kis = heads_ref((k.float().view(B, L, d) - kbar[:, None, :]).view(B * L, d), B, H, L)
    kis[:, :, L:] = kis[:, :, :L].mean(-1, keepdim=True)  # a real scale on the keys past L: only the mask keeps them out
    vt, vs = vt_ref(v, B, H, L)
    Q, K = Slab(qi, f["q"]), Slab(ki, f["k"])
    out = Slab(torch.zeros(B * L, d, device="cuda", dtype=BF), f["out"])
    scales = [_flat(t) for t in (qis, kis, vt.view(torch.float8_e4m3fn), vs)]
    (_, qsv), (_, ksv), (_, vtv), (_, vsv) = scales
    kw, maps = {}, []
    if tm is not None:
        maps = [_flat(t) for t in upload_maps(tm)]
        assert tuple(m.shape[2] for _, m in maps) == f["bh"]
        kw["bh_maps"] = (maps[0][1], maps[1][1])
    elif tiles is not None:
        kw["tiles"] = S.tile_map(*f["tiles"], "cuda")
    ops.attention_int8qk(Q.v, qsv, K.v, ksv, vtv, vsv, out.v, B, H, L, scale=f["scale"], **kw)
    compact = torch.empty(B * L, d, device="cuda", dtype=BF)
    ops.attention_int8qk(qi, qis, ki, kis, vt.view(torch.float8_e4m3fn), vs, compact, B, H, L, scale=f["scale"], **kw)
    torch.cuda.synchronize()
    for s in [Q, K, out] + [s for s, _ in scales + maps]:
        s.check("attention_int8qk")
    _exact(out.v, compact, "attention_int8qk: the strided launch against a compact one")
    del qi, ki, vt, scales, Q, K, compact
    want = _attention_ref(q, k, v, B, H, L, L, f["scale"], mask)
    chain = _attention_ref(q, k, v, B, H, L, L, f["scale"], mask, chain="int8")
    form = "per-(batch, head)" if tm is not None else "window" if tiles is not None else "dense"
    result, ratio = _fp8_verdict(out.v, want, chain, B, H, L, planted, f"attention_int8qk, {form}")
    return f"{form}: {result}", ratio


CHECKS_ALL = dict(CHECKS, **{name: globals()["check_" + name] for name in INT8_OPS})


def test_every_int8_b1_launch_matches_fp32(launches):
    from scail_b200 import ops
    failures, worst = [], {}
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    print(f"\n{len(launches)} distinct launches")
    for i, (name, f) in enumerate(launches):
        what = _describe(name, f)
        g = torch.Generator(device="cuda").manual_seed(3000 + i)
        try:
            result, ratio = CHECKS_ALL[name](ops, f, g)
            worst[name] = max(worst.get(name, 0.0), ratio)
            print(f"{what}: {result}")
        except AssertionError as e:
            print(f"FAIL {what}: {e}")
            failures.append(f"{what}: {e}")
        torch.cuda.empty_cache()
    print("worst |d|/bound per op (fp8 / int8 attention: worst block / (2 x chain's worst block + 1e-3); 0 = bit-exact): " +
          ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    print(f"{len(launches)} launches checked in {time.time() - t0:.0f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert not failures, f"{len(failures)} of {len(launches)} launches failed:\n" + "\n".join(failures)


def test_cfg_cache_skip_launches_are_the_direct_b1_ones(workload):
    """The conditional-only step of CFGCache makes only launches the direct b = 1 forwards made (so the checks of those
    stand for it), and it does launch the b = 1 self-attention of its mode."""
    N = {geo: (1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4) for geo, (t, h, w) in GEOMETRIES.items()}
    attn = {"bf16": "attention", "int8": "attention_int8qk"}
    for (geo, cm), keys in workload["skip"].items():
        extra = keys - workload["b1"][geo]
        assert not extra, f"{geo}, {cm}: the skipped step launched {len(extra)} keys the direct b = 1 forwards did not: " + \
            "; ".join(_describe(n, dict(k)) for n, k in sorted(extra, key=str)[:5])
        assert any(n == attn[cm] and dict(k)["B"] == 1 and dict(k).get("L", dict(k).get("kv_len")) == N[geo] for n, k in keys)
        print(f"{geo}, {cm}: the skipped step's {len(keys)} launch keys are all among the direct b = 1 forwards'")


def test_recorded_launches_cover_the_int8_and_b1_cases(launches):
    from scail_b200 import ops

    def has(name, **want):
        return any(n == name and all(v(f[k]) if callable(v) else f[k] == v for k, v in want.items()) for n, f in launches)

    Ns = {geo: (1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4) for geo, (t, h, w) in GEOMETRIES.items()}
    grid = lambda geo: (GEOMETRIES[geo][0], GEOMETRIES[geo][1] // 2, GEOMETRIES[geo][2] // 2)
    window = lambda geo: (lambda t: t is not None and (t[0].T, t[0].H, t[0].W) == grid(geo) and t[1] == 2)
    is_none, is_set = (lambda v: v is None), (lambda v: v is not None)

    def int8(geo, B, **attn):
        N = Ns[geo]
        return (has("rmsnorm_rope_int8q", rows=B * N, L=N, slabs=(0, 5120), rope=grid(geo) + (0, 0, 0)) and
                has("quant_k_int8", B=B, H=40, L=N) and has("attention_int8qk", B=B, H=40, L=N, **attn))

    def b1(geo, mode):
        N = Ns[geo]
        one = dict(B=1, H=40)
        return {
            "bf16": lambda: has("attention", q_len=N, kv_len=N, **one),
            "fp8": lambda: has("attention_fp8", L=N, tiles=None, **one) and has("gemm_fp8", M=N),
            "window 2": lambda: has("attention_sparse", q_len=N, tiles=window(geo), **one),
            "window 2, fp8 attention": lambda: has("attention_fp8", L=N, tiles=window(geo), **one),
            "adaptive": lambda: has("attention_sparse_bh", L=N, **one) and has("tile_pool", L=N, fp8=False, **one),
            "adaptive, fp8": lambda: has("attention_fp8_sparse_bh", L=N, **one) and has("tile_pool", L=N, fp8=True, int8=False,
                                                                                         **one),
            "int8": lambda: int8(geo, 1, tiles=None, bh=None),
            "int8, window 2": lambda: int8(geo, 1, tiles=window(geo)),
            "int8, adaptive": lambda: int8(geo, 1, bh=is_set) and has("tile_pool", L=N, int8=True, **one),
            "int8, fp8 linears": lambda: int8(geo, 1, tiles=None, bh=None) and has("gemm_fp8", M=N),
        }[mode]()

    cases = {}
    for geo, N in Ns.items():
        cases[f"int8_qk dense, b = 2, at {geo}"] = int8(geo, 2, tiles=None, bh=None)
        cases[f"int8_qk window 2, b = 2, at {geo}"] = int8(geo, 2, tiles=window(geo), bh=None)
        cases[f"int8_qk adaptive, b = 2, at {geo}"] = (int8(geo, 2, tiles=None, bh=is_set) and
                                                      has("tile_pool", B=2, L=N, int8=True))
        cases[f"int8_qk dense with fp8 linears, b = 2, at {geo}"] = int8(geo, 2, tiles=None, bh=is_none) and \
            has("gemm_fp8", M=2 * N)
        for mode in B1_MODES:
            cases[f"b = 1 {mode} at {geo}"] = b1(geo, mode)
    assert has("gemm", M=Ns["512x512"], rows_per_batch=Ns["512x512"], epilogue=ops.EPI_BIAS_GATE_RES)
    print("\n" + "\n".join(f"{'ok' if ok else 'MISSING'}: {what}" for what, ok in cases.items()))
    assert all(cases.values()), [what for what, ok in cases.items() if not ok]


# ---------------------------------------------------------------- the whole path vs the fp32 oracle
def test_full_width_block_at_480x832_int8_vs_oracle():
    """One 14B-width block plus the embeddings and the final layer at latent 21x60x104 (N = 42 510), b = 2 (two different
    text contexts), bf16 linears, in int8_qk and in fp8 attention, against the fp32 oracle.  At the attention level the
    restated int8 chain measured 0.71-0.73x the fp8 chain's error, so the INT8 block may not be worse than the fp8 one."""
    import oracle.dit_oracle as O
    m = full_width_model(1, seed=5)
    x0, cond, uc = step_inputs(6, *GEOMETRIES["480x832"])
    x = torch.cat([x0, x0]).to(BF)
    ctx = torch.cat([uc["crossattn"], cond["crossattn"]])
    ref, pose, clip = cond["ref_concat"], cond["concat_smpl_render"], cond["image_clip_features"]
    ts = torch.full((2,), 500.0, device="cuda")
    ad = m.mixins["adaln_layer"]
    orig = ad.layer_forward
    cap, got = {}, {}

    def lf(hid, mask, **kw):
        o = orig(hid, mask, **kw)
        cap["block"] = o.clone()
        return o

    ad.layer_forward = lf
    with torch.no_grad():
        for mode in ("int8_qk", True):
            ad.fp8_attention = mode
            out = m(x, timesteps=ts, context=ctx, ref_concat=ref, concat_smpl_render=pose, image_clip_features=clip).float()
            got[mode] = (cap["block"].float(), out)
    torch.cuda.synchronize()
    sd = {k: v.float() for k, v in m.state_dict().items()}
    del m, ad, orig
    old_sdpa = O.sdpa
    O.sdpa = lambda q, k, v: sdpa_fp32_chunked(q, k, v) if q.dtype == torch.float32 else old_sdpa(q, k, v)
    try:
        with torch.no_grad(), torch.device("cuda"):
            want, hid = O.dit_forward(sd, x.float(), ts, ctx.float(), ref.float(), pose.float(), clip.float(), 40, 1,
                                      return_hidden=True)
            hid = hid[1]
    finally:
        O.sdpa = old_sdpa
    for b, branch in enumerate(("uncond", "cond")):
        e = {mode: (rel(blk[b], hid[b]), rel(out[b], want[b])) for mode, (blk, out) in got.items()}
        (i_blk, i_out), (f_blk, f_out) = e["int8_qk"], e[True]
        print(f"480x832 block, b = 2, {branch} branch vs the fp32 oracle: int8_qk block {i_blk:.3e} out {i_out:.3e} | fp8 "
              f"attention block {f_blk:.3e} out {f_out:.3e} | int8 / fp8: block {i_blk / f_blk:.3f} out {i_out / f_out:.3f}")
        assert i_blk <= f_blk and i_out <= f_out, (branch, e)
