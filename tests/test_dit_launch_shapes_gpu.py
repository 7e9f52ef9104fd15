"""The DiT kernels at the launches a SCAIL-14B sampler step makes, against fp32, element by element.

test_every_dit_launch_matches_fp32: a full-width DiffusionTransformer (5120 / 40 heads / 13824, text_dim 4096, two blocks,
random weights) runs sampler.sampler_step on latents 21x64x64 (N = 27 904), 21x60x104 (N = 42 510, ragged: 14 keys in the
last tile, n_ref = 1560) and 21x64x112 (N = 48 832, 64 keys in the last tile) with the CFG batch of two 512-token text
contexts, in bf16, with fp8 linears + fp8 attention, and with the window-2 block-sparse attention (bf16 and fp8); the
per-rank b = 1 forward of the 2-GPU CFG split at 21x64x112; and two steps of FirstBlockCache(inf) at the two ragged
geometries (the first computes, the second skips).  Also at every geometry the content-adaptive attention
AdaptiveTiles(0.9, max_tiles=40), in bf16 and with fp8 linears + fp8 attention; at the two ragged geometries
FirstBlockCache(order=1) and (order=2) over four steps with thresholds 0, 0, 0, inf (three computed steps fill the
forecast slots, the fourth skips and forecasts from 2 or 3 of them); and at 21x64x112 sampler.sample with UniPC(3) over
make_flow_timesteps(4) (predictor orders 1, 2, 2, 1, the corrector from the second step on).  Every DiT entry point of
scail_b200.ops is wrapped by kernel_check.recording; each distinct launch (shapes, row strides and slab offsets of every
operand, batch-row counts, epilogue, RoPE geometry, tile map, map strides, slot counts, ...) is re-run on fresh seeded data
with the recorded views inside wider buffers whose other elements are sentinels (checked bit for bit after the launch),
against an fp32 reference on the GPU (TF32 off), or a float64 / bit-exact restatement where the kernel promises one: tile
pooling against the float64 tile mean, tile selection against its float64 restatement (tests/adaptive_oracle.py) on the
kernel's own pooled tiles, the forecast kernels against tests/forecast_oracle.py at every slot index and every coefficient
pattern the cache can pass (dead slots full of NaN), and the UniPC step against test_unipc_gpu.step_ref at the recorded
coefficients (unread slots full of NaN).

Attention data can fail: q, k give scaled logits with std ~3, and planted keys dominate chosen rows of batch 0 (key 0, the
last valid key, keys on both sides of a 128-key tile edge, and for sparse maps a key in an unlisted tile, which must have no
effect, and one in a listed tile).  Where batch 0's last key tile overhangs into batch 1 (kv_len % 128 != 0), batch 0's last
query row gets a winning key among batch 1's first rows: the TMA box of that tile reads it and only the mask keeps it out.
A leaked mask or a skipped tile moves such a row by the scale of V, not by a rounding.  The last batch's last key tile has
nothing after it (TMA zero-fills the overhang, and a zero key's logit 0 is far below an ordinary row's max of ~ +13), so
where kv_len % 128 != 0 the last query row of batch B - 1 gets logits <= -40 at heads 0 and H - 1 (_plant_last_tile): a
leaked key past the end then takes the whole row.  Every view has 128 sentinel rows after it, so a whole tile read or
stored past its last row lands on sentinels.  The per-(batch, head) kernels run
under maps from a real select_tiles run that differ across heads and batch elements; in both batch elements, at heads 0,
H/2 and H - 1, a row gets a key in a tile its own map omits but the next head's map lists (no effect), and one in a tile
its map lists.

test_full_width_block_at_480x832_cfg_batch_vs_oracle: one full-width block plus the embeddings and the final layer at
21x60x104, b = 2 (two different text contexts), against oracle/dit_oracle.py in fp32 on the GPU, next to the
reference-style bf16 library chain."""
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from adaptive_oracle import select_reference
from forecast_oracle import apply_forecast_ref
from kernel_check import assert_close_bf16, measure, recording
from step_cache_oracle import apply_ref, indicator_sums, update_ref
from test_adaptive_attention_gpu import bh_dense, masked_chain_fp8_bh, pool_ref, upload_maps
from test_fp8_attention_gpu import qk_ref, vt_ref
from test_fp8_gpu import deq, quant_ref
from test_scale_gpu import sdpa_fp32_chunked
from test_sparse_attention_gpu import heads
from test_step_cache_forecast_gpu import sentinel_slots, slot_tensor
from test_step_cache_gpu import operands as step_cache_operands, scratch as step_cache_scratch
from test_unipc_gpu import sentinel as unipc_sentinel, step_ref

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn
BF = torch.bfloat16

OPS = ("gemm", "gemm_fp8", "quant_rows_fp8", "quant_vt_fp8", "ln_modulate", "rmsnorm_rope", "attention", "attention_sparse",
       "attention_fp8", "adaln_modulation", "silu", "timestep_embedding", "patchify", "unpatchify", "cfg_euler_", "cast_bf16",
       "step_cache_indicator", "step_cache_update", "step_cache_apply", "tile_pool", "select_tiles", "attention_sparse_bh",
       "attention_fp8_sparse_bh", "step_cache_update_slot", "step_cache_apply_forecast", "unipc_step_")
GEOMETRIES = {"512x512": (21, 64, 64), "480x832": (21, 60, 104), "512x896": (21, 64, 112)}
ADAPTIVE = (0.9, 40)  # AdaptiveTiles(mass, max_tiles) of the adaptive modes
MODES = {"bf16": dict(), "fp8": dict(fp8_linear=True, fp8_attention=True), "window 2": dict(attention_window=2),
         "window 2, fp8 attention": dict(attention_window=2, fp8_attention=True), "adaptive": dict(attention_adaptive=True),
         "adaptive, fp8": dict(attention_adaptive=True, fp8_linear=True, fp8_attention=True)}
CACHED = ("480x832", "512x896")
B1 = "512x896"
FORECAST_THRESHOLDS = (0.0, 0.0, 0.0, math.inf)  # three computed steps fill the slots, the fourth skips and forecasts
N_REF = {(1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4): (h // 2) * (w // 2) for t, h, w in GEOMETRIES.values()}

GELU_TANH_ABS = 2.0 ** -11  # tanh.approx slack, as in test_gemm_tiles_gpu.py
ATT_ELEM = dict(elem_rel=2.0 ** -7, elem_abs=2.0 ** -8)  # as test_sparse_attention_gpu.py: P enters PV as bf16, then the output
LOGIT_STD = 3.0


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


def full_width_model(num_layers, seed=3):
    """The 14B block width with random weights (std 0.02) and the 1-D parameters (biases, norms) perturbed, as test_scale_gpu."""
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


def step_inputs(seed, t, h, w):
    """x0 (fp32 [1, t, 16, h, w]) and the sampler's cond / uc: two different 512-token text contexts; one ref, pose and
    257-token CLIP input shared by both CFG branches."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    x0 = torch.randn(1, t, 16, h, w, generator=g).cuda()
    cond = dict(crossattn=r(1, 512, 4096), ref_concat=r(1, 1, 16, h, w), concat_smpl_render=r(1, t, 16, h // 2, w // 2),
                image_clip_features=r(1, 257, 1280))
    return x0, cond, dict(crossattn=r(1, 512, 4096))


# ---------------------------------------------------------------- recording
def _view(t):
    """(row stride, first column inside its row, whether rows of the buffer precede it) of a 2-D row-strided view."""
    ld, off = t.stride(0), t.storage_offset()
    return (ld, off % ld, off >= ld)


def _rope_geometry(cos):
    """(T, H, W, h_shift, w_shift, first row) of the RoPE tables `cos`, or None without RoPE.  rope.build_tables keeps one
    pair per geometry and shift; `cos` is one of them or, under context parallelism, a row slice of one (first row: the
    slice's offset into its base table)."""
    from scail_b200 import rope
    if cos is None:
        return None
    for key, (c, _) in rope._DEV_CACHE.items():
        if cos.untyped_storage().data_ptr() == c.untyped_storage().data_ptr():
            assert key[7:] == (0, 120, 10000.0), key  # the model's global_rope_H / W and theta
            row, rem = divmod(cos.storage_offset() - c.storage_offset(), c.stride(0))
            assert rem == 0 and cos.stride() == c.stride() and row + cos.shape[0] <= c.shape[0], "not a row slice of its table"
            return key[2:7] + (row,)
    raise AssertionError("RoPE tables that rope.build_tables did not make")


def _tile_key(tiles):
    """(geometry, window) of a frame-window tile map (scail_b200.sparse keeps one per geometry and window), or None."""
    from scail_b200 import sparse
    if tiles is None:
        return None
    for (g, window, _), m in sparse._CACHE.items():
        if m is tiles:
            return (g, window)
    raise AssertionError("a tile map that sparse.tile_map did not make")


def _fields(name, a):
    """The fields that select the kernel, its grid and its edges for one call (`a`: the bound arguments)."""
    if name in ("gemm", "gemm_fp8"):
        x, w, out, res, gate = a["a"], a["w"], a["out"], a["residual"], a["gate"]
        M, K = x.shape
        N = w.shape[0]
        fp32 = bool(a.get("out_fp32")) if out is None else out.dtype == torch.float32
        return dict(M=M, N=N, K=K, a=_view(x), ldw=w.stride(0), out=(N, 0, False) if out is None else _view(out), fp32=fp32,
                    bias=a["bias"] is not None, epilogue=a["epilogue"], gate=None if gate is None else _view(gate),
                    rows_per_batch=a["rows_per_batch"],
                    residual=None if res is None else "out" if out is not None and res.data_ptr() == out.data_ptr() else _view(res)), 1
    if name == "quant_rows_fp8":
        return dict(M=a["x"].shape[0], K=a["x"].shape[1], x=_view(a["x"])), 1
    if name == "quant_vt_fp8":
        return dict(B=a["B"], H=a["H"], L=a["L"], v=_view(a["v"])), 1
    if name == "ln_modulate":
        x, shift = a["x"], a["shift"]
        B, n_in, D = x.shape
        return dict(B=B, n_in=n_in, D=D, rows_out=n_in if a["rows_out"] is None else a["rows_out"], row_offset=a["row_offset"],
                    gamma=a["gamma"] is not None, beta=a["beta"] is not None, mod_stride=None if shift is None else shift.stride(0),
                    eps=float(a["eps"]), fp8=a["out_fp8"] is not None), 1
    if name == "rmsnorm_rope":
        buf, o8 = a["buf"], a["out_fp8"]
        return dict(rows=buf.shape[0], rows_per_batch=a["rows_per_batch"], D=a["D"], buf=_view(buf), width=buf.shape[1],
                    slabs=tuple(o for o, _ in a["slabs"]), rope=_rope_geometry(a["cos"]), eps=float(a["eps"]),
                    fp8=None if o8 is None else (_view(o8[0][0]), o8[0][1].shape[-1])), 1
    if name in ("attention", "attention_sparse"):
        L = a.get("L")
        q_len, kv_len = (L, L) if name == "attention_sparse" else (a["q_len"], a["kv_len"])
        return dict(B=a["B"], H=a["H"], q_len=q_len, kv_len=kv_len,
                    q_rows=q_len if a["q_batch_rows"] is None else a["q_batch_rows"],
                    kv_rows=kv_len if a["kv_batch_rows"] is None else a["kv_batch_rows"],
                    q=_view(a["q"]), k=_view(a["k"]), v=_view(a["v"]), out=_view(a["out"]), q_total=a["q"].shape[0],
                    kv_total=a["k"].shape[0], scale=float(a["scale"] or 1.0 / math.sqrt(128)), accumulate=bool(a["accumulate"]),
                    tiles=_tile_key(a["tiles"]) if name == "attention_sparse" else None), 1
    if name == "attention_fp8":
        return dict(B=a["B"], H=a["H"], L=a["L"], q=_view(a["q8"]), k=_view(a["k8"]), out=_view(a["out"]),
                    scale=float(a["scale"] or 1.0 / math.sqrt(128)), tiles=_tile_key(a["tiles"])), 1
    if name == "adaln_modulation":
        return dict(shape=tuple(a["emb"].shape)), 1
    if name in ("silu", "cast_bf16"):
        return dict(shape=tuple(a["x"].shape)), 1
    if name == "timestep_embedding":
        return dict(B=a["t"].shape[0], dim=a["dim"]), 1
    if name == "patchify":
        B, T, C, H, W = a["x"].shape
        return dict(B=B, Br=a["ref"].shape[0], Bp=a["pose"].shape[0], T=T, H=H, W=W, C=C), 1
    if name == "unpatchify":
        return dict(B=a["B"], T=a["T"], Hp=a["Hp"], Wp=a["Wp"]), 1
    if name == "cfg_euler_":
        return dict(shape=tuple(a["x"].shape), scale=float(a["scale"]), dsigma=float(a["dsigma"])), 1
    if name == "step_cache_indicator":
        return dict(shape=tuple(a["h1"].shape), n_ref=a["n_ref"], n_seq=a["h1c"].shape[1]), 1
    if name in ("step_cache_update", "step_cache_apply"):
        return dict(shape=tuple(a["h"].shape), n_ref=a["n_ref"], n_seq=a["R"].shape[1]), 1
    if name == "tile_pool":
        xs = a["x_scale"]
        return dict(B=a["B"], H=a["H"], L=a["L"], x=_view(a["x"]), fp8=xs is not None, int8=a["x"].dtype == torch.int8,
                    L_pad=None if xs is None else xs.shape[-1]), 1
    if name == "select_tiles":
        return dict(B=a["B"], H=a["H"], L=a["L"], n_ref=a["n_ref"], mass=float(a["mass"]), max_tiles=a["max_tiles"],
                    ptr_stride=a["ptr"].shape[2], idx_stride=a["idx"].shape[2]), 1
    if name == "attention_sparse_bh":
        L = a["L"]
        return dict(B=a["B"], H=a["H"], L=L, q_rows=L if a["q_batch_rows"] is None else a["q_batch_rows"],
                    kv_rows=L if a["kv_batch_rows"] is None else a["kv_batch_rows"], q=_view(a["q"]), k=_view(a["k"]),
                    v=_view(a["v"]), out=_view(a["out"]), q_total=a["q"].shape[0], kv_total=a["k"].shape[0],
                    scale=float(a["scale"] or 1.0 / math.sqrt(128)), ptr_stride=a["ptr"].shape[2],
                    idx_stride=a["idx"].shape[2]), 1
    if name == "attention_fp8_sparse_bh":
        return dict(B=a["B"], H=a["H"], L=a["L"], q=_view(a["q8"]), k=_view(a["k8"]), out=_view(a["out"]),
                    L_pad=a["q_scale"].shape[-1], scale=float(a["scale"] or 1.0 / math.sqrt(128)),
                    ptr_stride=a["ptr"].shape[2], idx_stride=a["idx"].shape[2]), 1
    if name in ("step_cache_update_slot", "step_cache_apply_forecast"):
        # the slot index and the coefficients live on the device: the check runs every value of them
        R = a["R_slots"]
        return dict(shape=tuple(a["h"].shape), n_ref=a["n_ref"], n_seq=R.shape[2], n_slots=R.shape[0],
                    slot_stride=R[0].numel()), 1
    if name == "unipc_step_":
        coef = tuple(float(c) for c in a["coef"])
        return dict(shape=tuple(a["x"].shape), n_slots=a["slots"].shape[0], slot_stride=a["slots"].stride(0),
                    write_slot=int(a["write_slot"]), correct=bool(a["correct"]), active=tuple(c != 0.0 for c in coef),
                    coef=coef, scale=float(a["scale"]), sigma=float(a["sigma"])), 1
    raise KeyError(name)


@pytest.fixture(scope="module")
def launches():
    """[(op, key)] of every distinct DiT launch of the cases in the module docstring, in first-call order."""
    from scail_b200 import dit, ops, sampler, sparse
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    m = full_width_model(2)
    ad = m.mixins["adaln_layer"]
    sig = sampler.make_flow_timesteps(50, 5.0)
    with torch.no_grad(), recording(ops, OPS, _fields) as seen:
        for i, (geo, (t, h, w)) in enumerate(GEOMETRIES.items()):
            x0, cond, uc = step_inputs(10 + i, t, h, w)
            for mode in MODES.values():
                ad.fp8_linear, ad.fp8_attention = mode.get("fp8_linear", False), mode.get("fp8_attention", False)
                ad.attention_window = mode.get("attention_window")
                ad.attention_adaptive = sparse.AdaptiveTiles(*ADAPTIVE) if mode.get("attention_adaptive") else None
                sampler.sampler_step(m, x0.clone(), sig[0], sig[1], cond, uc, 4.0)
            ad.fp8_linear = ad.fp8_attention = False
            ad.attention_window = ad.attention_adaptive = None
            if geo in CACHED:  # the first step computes, the second skips: indicator, update and apply all launch
                c, x = FirstBlockCache(math.inf), x0.clone()
                sampler.sampler_step(m, x, sig[0], sig[1], cond, uc, 4.0, step_cache=c)
                sampler.sampler_step(m, x, sig[1], sig[2], cond, uc, 4.0, step_cache=c)
                assert [s for _, s in c.history] == [False, True]
                del c
                for order in (1, 2):  # computed steps write slots 0, 1, 0 (order 1) or 0, 1, 2; the skip reads 2 or 3
                    c, x = FirstBlockCache(0.0, order=order), x0.clone()
                    for j, threshold in enumerate(FORECAST_THRESHOLDS):
                        c.threshold = threshold
                        sampler.sampler_step(m, x, sig[j], sig[j + 1], cond, uc, 4.0, step_cache=c)
                    assert [s for _, s in c.history] == [False, False, False, True]
                    assert sum(cf != 0.0 for cf in c.buffers.ctl_coef.tolist()) == order + 1
                    del c
            if geo == B1:  # one rank of the 2-GPU CFG split: the conditional branch alone
                m(x0, timesteps=torch.full((1,), float(sig[0]) * 1000.0, device="cuda"), context=cond["crossattn"],
                  ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
                  image_clip_features=cond["image_clip_features"])
                # UniPC(3) over make_flow_timesteps(4): predictor orders 1, 2, 2, 1; the corrector on from the second step
                sampler.sample(m, x0.clone(), cond, uc, num_steps=4, solver=UniPC(3))
    torch.cuda.synchronize()
    del m, ad
    dit._WS.bufs.clear()
    torch.cuda.empty_cache()
    return [(name, dict(k)) for (name, k) in seen]


# ---------------------------------------------------------------- buffers with sentinels
_SENTINEL_BITS = {1: 0x7E, 2: 0x4680, 4: 0x46800000, 8: 0x40D0000000000000}  # e4m3 448 / int8 126, bf16, fp32, fp64 16384
_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
TRAILING = 128  # sentinel rows after a Slab's view: a whole 128-row tile read or stored past its last row lands on them


def _bits(t):
    return t.view(_INT[t.element_size()])


class Slab:
    """`data` [rows, cols] placed as a view at a recorded place (row stride, first column, rows before) of a wider buffer
    with TRAILING rows after it; every other element of the buffer is a sentinel, which check() asserts is unchanged."""

    def __init__(self, data, view):
        ld, c0, before = view
        rows, cols = data.shape
        self.r0, self.c0, self.rows, self.cols = (2 if before else 0), c0, rows, cols
        self.parent = torch.empty(self.r0 + rows + TRAILING, ld, device=data.device, dtype=data.dtype)
        _bits(self.parent).fill_(_SENTINEL_BITS[data.element_size()])
        self.v = self.parent[self.r0:self.r0 + rows, c0:c0 + cols]
        _bits(self.v).copy_(_bits(data))
        self.snap = _bits(self.parent).clone()

    def check(self, what):
        changed = _bits(self.parent) != self.snap
        changed[self.r0:self.r0 + self.rows, self.c0:self.c0 + self.cols] = False
        assert not changed.any(), f"{what}: {int(changed.sum())} sentinel elements beside the view were written"


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(BF)


def _zeros8(*shape):
    return torch.zeros(*shape, device="cuda", dtype=torch.uint8).view(FP8)


def _exact(got, want, what):
    assert torch.equal(_bits(got), _bits(want)), f"{what}: not bit-exact ({int((_bits(got) != _bits(want)).sum())} differ)"
    return "exact"


def _report(c):
    return f"rel-L2 {c.rel_l2:.2e}, worst |d|/bound {c.worst_ratio:.2f} at {c.worst_index}"


# ---------------------------------------------------------------- one launch vs fp32
def check_gemm(ops, f, g, fp8=False):
    M, N, K, epi = f["M"], f["N"], f["K"], f["epilogue"]
    a = _rand(g, M, K)
    w = _rand(g, N, K, scale=K ** -0.5)
    bias = _rand(g, N) if f["bias"] else None
    if fp8:  # operands in the e4m3 row format (quant_ref: the restatement test_fp8_gpu.py pins the kernel to)
        (aq, sa), (wq, sw) = quant_ref(a), quant_ref(w)
        A, W = Slab(aq, f["a"]), Slab(wq, (f["ldw"], 0, False))
        acc = deq(aq, sa) @ deq(wq, sw).T
    else:
        A, W = Slab(a, f["a"]), Slab(w, (f["ldw"], 0, False))
        acc = a.float() @ w.float().T
    del a, w
    if bias is not None:
        acc += bias.float()
    slabs, kw = [A, W], {}
    res = _rand(g, M, N) if f["residual"] is not None else None
    out = Slab(res if f["residual"] == "out" else torch.zeros(M, N, device="cuda", dtype=torch.float32 if f["fp32"] else BF),
               f["out"])
    slabs.append(out)
    if f["residual"] is not None:
        if f["residual"] == "out":
            kw["residual"] = out.v
        else:
            R = Slab(res, f["residual"])
            slabs.append(R)
            kw["residual"] = R.v
    elem_abs = 2.0 ** -12
    if epi == ops.EPI_BIAS_GATE_RES:
        rpb = f["rows_per_batch"]
        G = Slab(_rand(g, -(-M // rpb), N), f["gate"])
        slabs.append(G)
        kw.update(gate=G.v, rows_per_batch=rpb)
        want = res.float().addcmul_(G.v.float().repeat_interleave(rpb, 0)[:M], acc)
    elif epi == ops.EPI_BIAS_RES:
        want = acc.add_(res.float())
    elif epi == ops.EPI_BIAS_GELU:
        want, elem_abs = F.gelu(acc, approximate="tanh"), GELU_TANH_ABS
    elif epi == ops.EPI_BIAS_GELU_ERF:
        want = F.gelu(acc)
    elif epi == ops.EPI_BIAS_SILU:
        want = F.silu(acc)
    else:
        want = acc
    del acc
    if fp8:
        ops.gemm_fp8(A.v, sa, W.v, sw, bias, out=out.v, epilogue=epi, **kw)
    else:
        ops.gemm(A.v, W.v, bias, out=out.v, epilogue=epi, **kw)
    torch.cuda.synchronize()
    for s in slabs:
        s.check("gemm")
    if f["fp32"]:  # no rounding at all: only the fp32 summation order differs (as test_gemm_tiles_gpu.py)
        c = measure(out.v, want, elem_rel=0.0, elem_abs=2.0 ** -16)
        assert c.n_bad == 0, f"fp32 output: {c}"
        return _report(c), c.worst_ratio
    c = assert_close_bf16(out.v, want, "gemm", elem_abs=elem_abs)
    return _report(c), c.worst_ratio


def check_gemm_fp8(ops, f, g):
    return check_gemm(ops, f, g, fp8=True)


def check_quant_rows_fp8(ops, f, g):
    x = _rand(g, f["M"], f["K"], scale=3.0)
    x[f["M"] // 2] = 0  # an all-zero row: scale 1
    X = Slab(x, f["x"])
    q, s = ops.quant_rows_fp8(X.v)
    torch.cuda.synchronize()
    X.check("quant_rows_fp8 input")
    qr, sr = quant_ref(x)
    _exact(s, sr, "quant_rows_fp8 scales")
    return _exact(q, qr, "quant_rows_fp8 codes"), 0.0


def check_quant_vt_fp8(ops, f, g):
    B, H, L = f["B"], f["H"], f["L"]
    v = _rand(g, B * L, H * 128)
    V = Slab(v, f["v"])
    Lp = ops.fp8_pad(L)
    vt = torch.full((B, H, 128, Lp), 0x7F, device="cuda", dtype=torch.uint8).view(FP8)  # NaN everywhere before
    sc = torch.empty(B, H, 128, device="cuda")
    ops.quant_vt_fp8(V.v, B, H, L, vt, sc)
    torch.cuda.synchronize()
    V.check("quant_vt_fp8 input")
    want, ws = vt_ref(v, B, H, L)
    _exact(sc, ws, "quant_vt_fp8 scales")
    return _exact(vt.view(torch.uint8), want, "quant_vt_fp8 codes"), 0.0


def check_ln_modulate(ops, f, g):
    B, n_in, D, rows, off, eps = f["B"], f["n_in"], f["D"], f["rows_out"], f["row_offset"], f["eps"]
    x = _rand(g, B, n_in, D, scale=2.0) + _rand(g, B, n_in, 1)  # rows with a mean of their own
    kw = dict(eps=eps, rows_out=rows, row_offset=off)
    if f["gamma"]:
        kw["gamma"] = 1 + _rand(g, D, scale=0.1)
    if f["beta"]:
        kw["beta"] = _rand(g, D, scale=0.1)
    if f["mod_stride"] is not None:  # shift, scale: rows of the block's adaLN vectors (mod[:, k], stride 6 d) or [B, d]
        ms = f["mod_stride"]
        mod = _rand(g, B, ms, scale=0.5)
        if ms >= 2 * D:
            kw.update(shift=mod[:, :D], scale=mod[:, D:2 * D])
        else:
            kw.update(shift=_rand(g, B, D, scale=0.5), scale=_rand(g, B, D, scale=0.5))
        assert kw["shift"].stride(0) == ms
    want = F.layer_norm(x[:, off:off + rows].float(), (D,), None if not f["gamma"] else kw["gamma"].float(),
                        None if not f["beta"] else kw["beta"].float(), eps)
    if "shift" in kw:
        want = want * (1 + kw["scale"].float()[:, None]) + kw["shift"].float()[:, None]
    out = Slab(torch.zeros(B * rows, D, device="cuda", dtype=BF), (D, 0, True))
    ops.ln_modulate(x, out=out.v.view(B, rows, D), **kw)
    torch.cuda.synchronize()
    out.check("ln_modulate")
    c = assert_close_bf16(out.v.view(B, rows, D), want, "ln_modulate")
    if f["fp8"]:  # bit for bit quant_rows_fp8 of the bf16 result
        q = Slab(_zeros8(B * rows, D), (D, 0, True))
        s = Slab(torch.zeros(B * rows, 1, device="cuda"), (1, 0, True))
        ops.ln_modulate(x, out_fp8=(q.v, s.v.view(-1)), **kw)
        torch.cuda.synchronize()
        q.check("ln_modulate fp8 codes"), s.check("ln_modulate fp8 scales")
        qr, sr = quant_ref(out.v)
        _exact(s.v.view(-1), sr, "ln_modulate fp8 scales")
        _exact(q.v, qr, "ln_modulate fp8 codes")
        return _report(c) + "; fp8 form exact", c.worst_ratio
    return _report(c), c.worst_ratio


def _rotate_half(x):
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack((-x2, x1), -1).flatten(-2)


def check_rmsnorm_rope(ops, f, g):
    from scail_b200 import rope
    rows, rpb, D, eps = f["rows"], f["rows_per_batch"], f["D"], f["eps"]
    data = _rand(g, rows, f["width"], scale=2.0)
    weights = [1 + _rand(g, D, scale=0.1) for _ in f["slabs"]]
    slabs = list(zip(f["slabs"], weights))
    cos = sin = None
    if f["rope"] is not None:  # the geometry's real tables (shifted, and the recorded row slice of them)
        *geo, row = f["rope"]
        cos, sin = rope.build_tables("cuda", 128, *geo)
        assert row + rpb <= cos.shape[0]
        cos, sin = cos[row:row + rpb], sin[row:row + rpb]
    buf = Slab(data, f["buf"])
    ops.rmsnorm_rope(buf.v, rpb, D, slabs, cos, sin, eps=eps)
    torch.cuda.synchronize()
    buf.check("rmsnorm_rope")
    other = torch.ones(f["width"], dtype=torch.bool)
    worst, reports = 0.0, []
    for o, wgt in slabs:
        other[o:o + D] = False
        x = data[:, o:o + D].float()
        y = wgt.float() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))  # oracle rmsnorm: g * (x * rstd)
        if cos is not None:  # oracle RoPE on interleaved pairs, token = first row + row % rows_per_batch of the base table
            tok = torch.arange(rows, device="cuda") % rpb
            yh = y.view(rows, D // 128, 128)
            y = (yh * cos[tok][:, None] + _rotate_half(yh) * sin[tok][:, None]).view(rows, D)
        c = assert_close_bf16(buf.v[:, o:o + D], y, f"rmsnorm_rope slab at column {o}")
        worst = max(worst, c.worst_ratio)
        reports.append(_report(c))
    _exact(buf.v[:, other.cuda()], data[:, other.cuda()], "rmsnorm_rope columns outside the slabs")
    if f["fp8"] is not None:  # bit for bit qk_ref of the bf16 result; the buffer itself is only read
        view8, Lp = f["fp8"]
        B, H = rows // rpb, D // 128
        src = Slab(data, f["buf"])
        outs = [(Slab(_zeros8(rows, D), view8), torch.full((B, H, Lp), 7.0, device="cuda"))
                for _ in slabs]
        ops.rmsnorm_rope(src.v, rpb, D, slabs, cos, sin, eps=eps, out_fp8=[(q.v, s) for q, s in outs])
        torch.cuda.synchronize()
        src.check("rmsnorm_rope fp8 input")
        _exact(src.v, data, "rmsnorm_rope fp8 form: its input")
        for (o, _), (q, s) in zip(slabs, outs):
            q.check("rmsnorm_rope fp8 codes")
            qr, sr = qk_ref(buf.v[:, o:o + D], B, H, rpb)
            _exact(s, sr, "rmsnorm_rope fp8 scales")
            _exact(q.v, qr, "rmsnorm_rope fp8 codes")
        reports.append("fp8 form exact")
    return "; ".join(reports), worst


# ---------------------------------------------------------------- attention
def _tile_matrix(key):
    """bool [n_q_tiles, n_kv_tiles] on the GPU of a recorded (geometry, window), and the host map."""
    from scail_b200 import sparse
    ptr, idx, _ = sparse.frame_window_tiles(*key)
    n = len(ptr) - 1
    rows = torch.repeat_interleave(torch.arange(n), torch.from_numpy(ptr[1:] - ptr[:-1]).long())
    t = torch.zeros(n, n, dtype=torch.bool)
    t[rows, torch.from_numpy(idx).long()] = True
    return t.cuda()


def _attention_ref(q, k, v, B, H, q_len, kv_len, scale, tiles=None, chain=False):
    """fp32 softmax(scale q k^T) v per batch and head over [B * len, H * 128] operands, queries chunked; tiles: the key tiles
    each 128-query tile may see, bool [n_q_tiles, n_kv_tiles] for every (batch, head) or [B, H, n_q_tiles, n_kv_tiles] per
    (batch, head).  chain: the restated fp8 chain of test_fp8_attention_gpu.chain_fp8 (dequantised per-token Q, K and
    per-channel V, P^ = e4m3(2^8 p) against the row max over the allowed keys, l the sum of the unquantised 2^8 p); chain=
    "int8": the int8-QK chain of test_int8qk_attention_gpu.chain_int8 (Q and K' = K - its fp64 per-(batch, channel) mean
    over the kv_len keys in the INT8 row format, V and P as in the fp8 chain)."""
    from test_int8qk_attention_gpu import int8_ref
    out = torch.empty(B * q_len, H * 128, device="cuda")
    chunk = min(4096, max(128, (2 ** 29 // (H * kv_len)) // 128 * 128))
    for b in range(B):
        heads = lambda x, n: x[b * n:(b + 1) * n].float().view(n, H, 128).transpose(0, 1)
        qh, kh, vh = heads(q, q_len), heads(k, kv_len), heads(v, kv_len)
        if chain == "int8":
            qh = deq(*int8_ref(qh.reshape(-1, 128))).view(H, q_len, 128)
            kh = kh - kh.double().mean(1, keepdim=True).float()
            kh = deq(*int8_ref(kh.reshape(-1, 128))).view(H, kv_len, 128)
        elif chain:
            qh = deq(*quant_ref(qh.reshape(-1, 128))).view(H, q_len, 128)
            kh = deq(*quant_ref(kh.reshape(-1, 128))).view(H, kv_len, 128)
        if chain:
            vh = deq(*quant_ref(vh.transpose(1, 2).reshape(-1, kv_len))).view(H, 128, kv_len).transpose(1, 2)
        kt = kh.transpose(1, 2)
        for i in range(0, q_len, chunk):
            s = (qh[:, i:i + chunk] @ kt) * scale
            if tiles is not None:  # s: [H, rows, kv_len]
                qt = torch.arange(i, i + s.shape[1], device="cuda") // 128
                allowed = (tiles[qt] if tiles.dim() == 2 else tiles[b][:, qt]).repeat_interleave(128, -1)[..., :kv_len]
                s.masked_fill_(~(allowed if allowed.dim() == 3 else allowed[None]), float("-inf"))
            if chain:
                p = torch.exp(s - s.amax(-1, keepdim=True)) * 256.0
                o = (p.to(FP8).float() @ vh) / p.sum(-1, keepdim=True)
            else:
                o = torch.softmax(s, -1) @ vh
            out[b * q_len + i:b * q_len + i + s.shape[1]] = o.transpose(0, 1).reshape(s.shape[1], H * 128)
            del s, o
    return out


def _attention_data(g, f, tiles=None):
    """q, k, v bf16 [B * len, H * 128] with scaled logits of std ~3 and planted keys (module docstring), and where kv_len %
    128 != 0 the last-tile plant of _plant_last_tile.  -> (q, k, v, [(global query row, head, whether the row may see its
    planted key)])."""
    B, H, q_len, kv_len = f["B"], f["H"], f["q_len"], f["kv_len"]
    s = LOGIT_STD ** 0.5
    q, k, v = _rand(g, B * q_len, H * 128, scale=s), _rand(g, B * kv_len, H * 128, scale=s), _rand(g, B * kv_len, H * 128)
    n_kt = -(-kv_len // 128)
    edge = 128 * (n_kt // 2)
    plants = [(3, kv_len - 1, 0.5), (q_len - 2, 0, 0.5), (q_len // 2, edge - 1, 0.5), (q_len // 2 + 1, edge, 0.5)]
    if B > 1 and kv_len % 128:  # batch 0's last key tile overhangs into batch 1: its key 5 is inside that TMA box
        plants.append((q_len - 1, kv_len + 5, 1.0))
    if kv_len > q_len and kv_len % q_len == 0:  # context parallelism: local queries against P = kv_len / q_len gathered shards
        # the first and last key of every shard; where a shard boundary falls inside a 128-key tile, those are its two sides
        keys = sorted({key for p in range(kv_len // q_len) for key in (p * q_len, (p + 1) * q_len - 1)})
        plants += [(10 + 17 * j, key, 0.5) for j, key in enumerate(keys)]
    if tiles is not None:  # a key in a tile the row's map does not list (no effect), and one in a listed tile
        t = tiles.shape[0] // 2
        listed = torch.nonzero(tiles[t]).flatten().tolist()
        unlisted = torch.nonzero(~tiles[t]).flatten().tolist()
        assert unlisted, "a window-2 map that lists every tile"
        plants += [(128 * t + 5, 128 * unlisted[len(unlisted) // 2] + 7, 1.0), (128 * t + 6, 128 * listed[-1] + 9, 0.5)]
    rows = []
    for row, key, alpha in plants:
        visible = key < kv_len and (tiles is None or bool(tiles[row // 128, key // 128]))
        for h in (0, H - 1):
            c = slice(h * 128, h * 128 + 128)
            q[row, c] = (alpha * k[key, c].float()).to(BF)
            rows.append((row, h, visible))
    if kv_len % 128:
        rows += _plant_last_tile(g, q, k, B, H, q_len, kv_len, f.get("scale") or 128 ** -0.5, B > 1)
    return q, k, v, rows


def _plant_last_tile(g, q, k, B, H, q_len, kv_len, scale, overhang):
    """The last query row of batch B - 1, at heads 0 and H - 1, sees only logits <= -40: one common vector u is added to
    every key of that (batch, head) and the row's q = -gamma u.  Softmax is shift-invariant per row, so only that row's
    expected output changes, and it stays an ordinary row (its logits still spread by ~3).  The key tile past batch B - 1's
    last key overhangs the end of the operand: TMA zero-fills it, and a zero key gets logit 0.  Without the mask those keys
    take practically all of the row's weight and move it by its whole norm; with ordinary logits (max ~ +13) they would
    carry ~1e-4 of it, below one bf16 rounding.  INT8 smoothing subtracts u again (mean-centred logits of a row cannot all
    be negative), so for attention_int8qk this row is ordinary; there batch 0's overhang plant and the K scales past L
    (check_attention_int8qk) test the mask.  overhang: batch 0's last row was planted with batch 1's key 5, so u is kept
    orthogonal to that key (its winning logit stays as it was).  -> [(global row, head, False)]."""
    row, rows = (B - 1) * q_len + q_len - 1, []
    for h in (0, H - 1):
        c = slice(h * 128, h * 128 + 128)
        keys = k[(B - 1) * kv_len:B * kv_len, c]
        u = torch.randn(128, device="cuda", generator=g) * 4.0
        if overhang:
            w = k[kv_len + 5, c].float()
            u -= (u @ w) / (w @ w) * w
        keys.copy_((keys.float() + u).to(BF))
        ub = u.to(BF).float()
        least = float((keys.float() @ ub).min())  # min over the keys of u . k, > 0: |u|^2 ~ 2048 against |u . k| ~ 80
        assert least > 0, least
        gamma = 2.0 ** math.ceil(math.log2(40.0 / (scale * least)))  # a power of two: q = -gamma u is exact in bf16
        q[row, c] = (-gamma * ub).to(BF)
        rows.append((row, h, False))
    return rows


def _block_rel(got, want, B, H, L):
    """rel-L2 of every (batch, head, 128-query tile) block: [B, n_tiles, H]."""
    n = -(-L // 128)
    d = (got.float() - want).pow(2).view(B, L, H, 128).sum(-1)
    w = want.pow(2).view(B, L, H, 128).sum(-1)
    pad = lambda x: F.pad(x, (0, 0, 0, n * 128 - L)).view(B, n, 128, H).sum(2)
    return (pad(d) / pad(w)).sqrt()


def check_attention(ops, f, g, sparse=False):
    from scail_b200 import sparse as S
    B, H, q_len, kv_len = f["B"], f["H"], f["q_len"], f["kv_len"]
    assert f["q_rows"] == q_len and f["kv_rows"] == kv_len and f["q_total"] == B * q_len and f["kv_total"] == B * kv_len
    tiles = _tile_matrix(f["tiles"]) if sparse else None
    q, k, v, planted = _attention_data(g, f, tiles)
    Q, K, V = Slab(q, f["q"]), Slab(k, f["k"]), Slab(v, f["v"])
    before = _rand(g, B * q_len, H * 128) if f["accumulate"] else torch.zeros(B * q_len, H * 128, device="cuda", dtype=BF)
    out = Slab(before, f["out"])
    if sparse:
        ops.attention_sparse(Q.v, K.v, V.v, out.v, B, H, q_len, S.tile_map(*f["tiles"], "cuda"), scale=f["scale"],
                             accumulate=f["accumulate"])
    else:
        ops.attention(Q.v, K.v, V.v, out.v, B, H, q_len, kv_len, scale=f["scale"], accumulate=f["accumulate"])
    torch.cuda.synchronize()
    for s in (Q, K, V, out):
        s.check("attention")
    want = _attention_ref(q, k, v, B, H, q_len, kv_len, f["scale"], tiles)
    if f["accumulate"]:
        want += before.float()
    c = assert_close_bf16(out.v, want, "attention", **ATT_ELEM)
    return _report(c) + f", {len(planted)} planted rows", c.worst_ratio


def check_attention_sparse(ops, f, g):
    return check_attention(ops, f, g, sparse=True)


def check_attention_fp8(ops, f, g):
    from scail_b200 import sparse as S
    B, H, L = f["B"], f["H"], f["L"]
    tiles = _tile_matrix(f["tiles"]) if f["tiles"] is not None else None
    q, k, v, planted = _attention_data(g, dict(B=B, H=H, q_len=L, kv_len=L), tiles)
    (q8, qs), (k8, ks), (vt, vs) = qk_ref(q, B, H, L), qk_ref(k, B, H, L), vt_ref(v, B, H, L)
    Q, K = Slab(q8, f["q"]), Slab(k8, f["k"])
    out = Slab(torch.zeros(B * L, H * 128, device="cuda", dtype=BF), f["out"])
    m = S.tile_map(*f["tiles"], "cuda") if f["tiles"] is not None else None
    ops.attention_fp8(Q.v, qs, K.v, ks, vt.view(FP8), vs, out.v, B, H, L, scale=f["scale"], tiles=m)
    torch.cuda.synchronize()
    for s in (Q, K, out):
        s.check("attention_fp8")
    want = _attention_ref(q, k, v, B, H, L, L, f["scale"], tiles)
    chain = _attention_ref(q, k, v, B, H, L, L, f["scale"], tiles, chain=True)
    return _fp8_verdict(out.v, want, chain, B, H, L, planted, "attention_fp8")


def _fp8_verdict(got, want, chain, B, H, L, planted, what):
    """The e4m3 attention output got against the fp32 reference want, bounded by the restated fp8 chain's own error: overall
    rel-L2, the worst (batch, 128-query tile, head) block, and every planted row (global row, head, whether its key is
    visible)."""
    assert torch.isfinite(got.float()).all()
    e, e_chain = rel(got, want), rel(chain, want)
    assert e <= 1.25 * e_chain + 1e-3, f"{what}: rel-L2 {e:.3e} > 1.25 x chain {e_chain:.3e} + 1e-3"
    blk, blk_chain = _block_rel(got, want, B, H, L), _block_rel(chain, want, B, H, L)
    worst, worst_chain = float(blk.max()), float(blk_chain.max())
    at = tuple(int(i) for i in torch.unravel_index(blk.argmax(), blk.shape))
    assert worst <= 2 * worst_chain + 1e-3, (f"{what}: worst (batch, 128-query tile, head) block {at} rel-L2 {worst:.3e} "
                                             f"> 2 x the chain's worst block {worst_chain:.3e} + 1e-3")
    for row, h, visible in planted:
        # a visible planted key takes the whole weight: P^ = 2^8 there in both, so the row matches the chain closely.  A
        # masked one leaves an ordinary row, which differs from the chain by the chain's own roundings (~2e-2); had the key
        # leaked in, it would take the whole weight and move the row by the scale of V (rel-L2 ~1).
        c = slice(h * 128, h * 128 + 128)
        e_row, bound = rel(got[row, c], chain[row, c]), 1e-2 if visible else 0.1
        assert e_row < bound, (f"{what}: planted row {row}, head {h} ({'visible' if visible else 'masked'} key): "
                               f"rel-L2 vs the chain {e_row:.3e} >= {bound}")
    ratio = worst / (2 * worst_chain + 1e-3)
    return (f"rel-L2 {e:.2e} (chain {e_chain:.2e}); worst block {worst:.2e} at {at} vs chain's worst {worst_chain:.2e}: "
            f"block ratio {worst / worst_chain:.2f}, {len(planted)} planted rows"), ratio


# ---------------------------------------------------------------- content-adaptive attention
def _flat(data):
    """A Slab of a contiguous tensor taken as rows of its last dimension: two sentinel rows before it and TRAILING after it,
    and a view that is contiguous again.  -> (slab, the view in data's shape)."""
    s = Slab(data.reshape(-1, data.shape[-1]), (data.shape[-1], 0, True))
    return s, s.v.view(data.shape)


def check_tile_pool(ops, f, g):
    """Tile means against float64 within 1e-6 relative (as test_adaptive_attention_gpu), the ragged last tile included; in
    e4m3 or INT8 (the row format of test_int8qk_attention_gpu.heads_ref) the codes times per-(token, head) scales that
    differ from token to token, with NaN past L (never read)."""
    from test_int8qk_attention_gpu import heads_ref
    B, H, L = f["B"], f["H"], f["L"]
    n = -(-L // 128)
    x = _rand(g, B * L, H * 128, scale=2.0) + _rand(g, B * L, 1)  # rows with a mean of their own
    slabs = []
    if f["fp8"]:
        codes, sc = (heads_ref if f["int8"] else qk_ref)(x, B, H, L)
        assert sc.shape[-1] == f["L_pad"]
        sc[:, :, L:] = math.nan
        X = Slab(codes, f["x"])
        S, scale = _flat(sc)
        slabs.append(S)
        x64 = (codes.float().double().view(B, L, H, 128) * sc[:, :, :L].permute(0, 2, 1).double()[..., None]).view(B * L, H * 128)
    else:
        X, scale, x64 = Slab(x, f["x"]), None, x.double()
    O, out = _flat(torch.zeros(B, H, n, 128, device="cuda"))
    slabs += [X, O]
    ops.tile_pool(X.v, B, H, L, out, x_scale=scale)
    torch.cuda.synchronize()
    for s in slabs:
        s.check("tile_pool")
    del x
    want = pool_ref(x64, B, H, L)
    del x64
    ratio = float(((out.double() - want).abs() / (1e-6 * want.abs() + 1e-30)).max())
    assert ratio <= 1, f"tile_pool: worst |d| / (1e-6 |float64 mean|) = {ratio:.3g}"
    return f"worst |d| / (1e-6 |mean|) {ratio:.2f}; last tile {L - 128 * (n - 1)} rows", ratio


def _structured(g, B, L, H, amp=3.0):
    """test_adaptive_attention_gpu.structured() generated on the GPU: tiles that share a component of amplitude amp plus
    token noise (at B = 2, L = 48 832 the host version holds ~2 GB)."""
    d, n = H * 128, -(-L // 128)
    base = (torch.randn(B, n, 1, d, device="cuda", generator=g) * amp).expand(B, n, 128, d).reshape(B, n * 128, d)[:, :L]
    return (base + torch.randn(B, L, d, device="cuda", generator=g)).reshape(B * L, d).to(BF)


def _select(ops, f, qbar, kbar):
    """select_tiles at the recorded arguments into maps with sentinels around them -> (slabs, ptr, idx)."""
    B, H, L = f["B"], f["H"], f["L"]
    P, ptr = _flat(torch.zeros(B, H, f["ptr_stride"], device="cuda", dtype=torch.int32))
    I, idx = _flat(torch.zeros(B, H, f["idx_stride"], device="cuda", dtype=torch.int32))
    scratch = torch.empty(ops.select_scratch_len(B, H, L), device="cuda", dtype=torch.int32)
    ops.select_tiles(qbar, kbar, B, H, L, f["n_ref"], f["mass"], f["max_tiles"], ptr, idx, scratch)
    return [P, I], ptr, idx


def check_select_tiles(ops, f, g):
    """Maps chosen from the kernel's own pooled tiles of structured Q, K: every (b, h) map valid, the forced tiles (the
    diagonal and every tile holding a reference token) listed, and the rows equal to the float64 restatement except rows
    within rounding of their cutoff, which must stay <= 1e-3 of all rows (as test_adaptive_attention_gpu)."""
    B, H, L, n_ref = f["B"], f["H"], f["L"], f["n_ref"]
    n = -(-L // 128)
    q = _structured(g, B, L, H)
    Qb, qbar = _flat(ops.tile_pool(q, B, H, L))
    del q
    k = _structured(g, B, L, H)
    Kb, kbar = _flat(ops.tile_pool(k, B, H, L))
    del k
    slabs, ptr, idx = _select(ops, f, qbar, kbar)
    torch.cuda.synchronize()
    for s in [Qb, Kb] + slabs:
        s.check("select_tiles")
    got = bh_dense(ptr, idx).numpy()  # checks every (b, h) map with ops.check_tile_map
    n_ref_t = -(-n_ref // 128)
    missing = np.argwhere(~got[..., :n_ref_t])
    assert missing.size == 0, f"select_tiles: reference tiles not listed at (b, h, q tile, k tile) {missing[:5].tolist()}"
    assert got[..., np.arange(n), np.arange(n)].all(), "select_tiles: a diagonal tile not listed"
    want, near = select_reference(qbar.cpu().numpy(), kbar.cpu().numpy(), L, n_ref, f["mass"], f["max_tiles"], band=1e-5)
    diff = (got != want).any(-1)
    bad = np.argwhere(diff & ~near)
    assert bad.size == 0, f"select_tiles: {len(bad)} rows differ from the float64 restatement, e.g. (b, h, q tile) {bad[:5].tolist()}"
    assert near.mean() <= 1e-3, f"select_tiles: {near.mean():.2e} of the rows sit at their cutoff"
    return (f"density {got.mean():.3f}, {n_ref_t} reference tiles forced, {int(diff.sum())} of {diff.size} rows differ "
            f"(all within rounding of the cutoff, {int(near.sum())} rows there)"), 0.0


def _adaptive_data(ops, g, f):
    """q, k, v bf16 [B * L, H * 128] (logit std ~3), per-(b, h) maps tm (bool [B, H, n, n] on the host) from a real
    select_tiles run on q, k at the adaptive mode's settings, and planted keys -> (q, k, v, tm, [(global query row, head,
    whether the row may see its planted key)]).  In every batch element, at heads 0, H/2 and H - 1, a query tile gets a key
    in a tile its own map omits but the next head's map lists (no effect), and one in a listed tile (batch 0: the last
    valid key, in the ragged last tile); where batch 0's last key tile overhangs into batch 1, batch 0's last query row gets
    a winning key among batch 1's first rows (as _attention_data)."""
    B, H, L = f["B"], f["H"], f["L"]
    n = -(-L // 128)
    s = LOGIT_STD ** 0.5
    q, k, v = _rand(g, B * L, H * 128, scale=s), _rand(g, B * L, H * 128, scale=s), _rand(g, B * L, H * 128)
    sel = dict(B=B, H=H, L=L, n_ref=N_REF[L], mass=ADAPTIVE[0], max_tiles=ADAPTIVE[1], ptr_stride=n + 1, idx_stride=n * n)
    _, ptr, idx = _select(ops, sel, ops.tile_pool(q, B, H, L), ops.tile_pool(k, B, H, L))
    tm = bh_dense(ptr, idx)
    assert not torch.equal(tm[0, 0], tm[0, 1]) and (B == 1 or not torch.equal(tm[0, 0], tm[1, 0])), "maps that do not differ"
    plants = []
    for b in range(B):
        for j, h in enumerate((0, H // 2, H - 1)):
            t = (n // 3 + 5 * j + 11 * b) % n
            unlisted = [u for u in torch.nonzero(~tm[b, h, t]).flatten().tolist() if u != n - 1]
            u = unlisted[len(unlisted) // 2]
            w = n - 1 if b == 0 else unlisted[0]
            assert u != w
            tm[b, (h + 1) % H, t, u] = True  # another head's map lists the tile
            tm[b, h, t, w] = True
            plants += [(b, h, 128 * t + 5, 128 * u + 7, 1.0), (b, h, 128 * t + 6, L - 1 if w == n - 1 else 128 * w + 9, 0.5)]
            if b == 0 and B > 1 and L % 128:  # batch 1's key 5 lies inside batch 0's last key tile (listed: the diagonal)
                plants.append((0, h, L - 1, L + 5, 1.0))
    rows = []
    for b, h, row, key, alpha in plants:
        c = slice(h * 128, h * 128 + 128)
        q[b * L + row, c] = (alpha * k[b * L + key, c].float()).to(BF)
        rows.append((b * L + row, h, key < L and bool(tm[b, h, row // 128, key // 128])))
    return q, k, v, tm, rows


def check_attention_sparse_bh(ops, f, g):
    B, H, L = f["B"], f["H"], f["L"]
    assert f["q_rows"] == L and f["kv_rows"] == L and f["q_total"] == B * L and f["kv_total"] == B * L
    q, k, v, tm, planted = _adaptive_data(ops, g, f)
    Q, K, V = Slab(q, f["q"]), Slab(k, f["k"]), Slab(v, f["v"])
    out = Slab(torch.zeros(B * L, H * 128, device="cuda", dtype=BF), f["out"])
    maps = [_flat(t) for t in upload_maps(tm)]
    assert [m.shape[2] for _, m in maps] == [f["ptr_stride"], f["idx_stride"]]
    ops.attention_sparse_bh(Q.v, K.v, V.v, out.v, B, H, L, maps[0][1], maps[1][1], scale=f["scale"])
    torch.cuda.synchronize()
    for s in [Q, K, V, out] + [s for s, _ in maps]:
        s.check("attention_sparse_bh")
    want = _attention_ref(q, k, v, B, H, L, L, f["scale"], tm.cuda())
    c = assert_close_bf16(out.v, want, "attention_sparse_bh", **ATT_ELEM)
    return _report(c) + f", density {tm.float().mean():.3f}, {len(planted)} planted rows", c.worst_ratio


def check_attention_fp8_sparse_bh(ops, f, g):
    B, H, L = f["B"], f["H"], f["L"]
    assert f["scale"] == 1.0 / math.sqrt(128)  # masked_chain_fp8_bh's scale
    q, k, v, tm, planted = _adaptive_data(ops, g, f)
    (q8, qs), (k8, ks), (vt, vs) = qk_ref(q, B, H, L), qk_ref(k, B, H, L), vt_ref(v, B, H, L)
    assert qs.shape[-1] == f["L_pad"]
    Q, K = Slab(q8, f["q"]), Slab(k8, f["k"])
    scales = [_flat(t) for t in (qs, ks, vt.view(FP8), vs)]
    out = Slab(torch.zeros(B * L, H * 128, device="cuda", dtype=BF), f["out"])
    maps = [_flat(t) for t in upload_maps(tm)]
    assert [m.shape[2] for _, m in maps] == [f["ptr_stride"], f["idx_stride"]]
    (_, qsv), (_, ksv), (_, vtv), (_, vsv) = scales
    ops.attention_fp8_sparse_bh(Q.v, qsv, K.v, ksv, vtv, vsv, out.v, B, H, L, maps[0][1], maps[1][1], scale=f["scale"])
    torch.cuda.synchronize()
    for s in [Q, K, out] + [s for s, _ in scales + maps]:
        s.check("attention_fp8_sparse_bh")
    del q8, k8, vt, scales, Q, K
    tmc = tm.cuda()
    want = _attention_ref(q, k, v, B, H, L, L, f["scale"], tmc)
    chain = masked_chain_fp8_bh(heads(q, B, L, H), heads(k, B, L, H), heads(v, B, L, H), tmc, chunk=128)
    chain = chain.transpose(1, 2).reshape(B * L, H * 128)
    return _fp8_verdict(out.v, want, chain, B, H, L, planted, "attention_fp8_sparse_bh")


# ---------------------------------------------------------------- forecast cache and UniPC
def check_step_cache_update_slot(ops, f, g):
    """Every slot value -1 .. n_slots - 1 on the recorded [B, N, d] and slots: the named slot equals update_ref bit for bit;
    the others, NaN-patterned sentinels, keep their bits (slot -1: all of them)."""
    (B, N, d), n_ref, n_seq, n_slots = f["shape"], f["n_ref"], f["n_seq"], f["n_slots"]
    assert f["slot_stride"] == B * n_seq * d
    Hs, h = _flat(_rand(g, B, N, d, scale=4.0))
    Cs, h1c = _flat(_rand(g, B, n_seq, d))
    want = update_ref(h, h1c, n_ref)
    before = sentinel_slots(n_slots, B, n_seq, d)
    for s in range(-1, n_slots):
        Rs, R = _flat(before)
        ops.step_cache_update_slot(h, h1c, R, slot_tensor(s), n_ref)
        torch.cuda.synchronize()
        for slab in (Hs, Cs, Rs):
            slab.check(f"step_cache_update_slot, slot {s}")
        for k in range(n_slots):
            if k == s:
                _exact(R[k], want, f"step_cache_update_slot: slot {s}")
            else:
                _exact(R[k], before[k], f"step_cache_update_slot: slot {k} while writing slot {s}")
        del Rs, R
    return f"exact, slots -1 .. {n_slots - 1}, slot {n_slots - 1} ends {4 * n_slots * f['slot_stride'] / 2**30:.2f} GiB in", 0.0


def _forecast_patterns(n_slots):
    """(coefficients, the slot filled with NaN or None) for what the cache can pass: every slot active, one slot dead (its
    coefficient 0, its contents NaN: it must not be read), none active (h unchanged), and one slot at exactly 1 (which is
    step_cache_apply of that slot)."""
    out = [({2: [2.0, -1.0], 3: [3.0, -3.0, 1.0]}[n_slots], None)]  # linear and quadratic extrapolation, evenly spaced
    for dead in range(n_slots):
        c = [0.5, -1.25, 1.75][:n_slots]
        c[dead] = 0.0
        out.append((c, dead))
    out.append(([0.0] * n_slots, None))
    out += [([1.0 if k == s else 0.0 for k in range(n_slots)], None) for s in range(n_slots)]
    return out


def check_step_cache_apply_forecast(ops, f, g):
    """Bit for bit apply_forecast_ref for every coefficient pattern of _forecast_patterns (a coefficient past n_slots is NaN:
    never read); (1 at slot s) also equals step_cache_apply of slot s; the ref and pose rows and the slots are untouched."""
    (B, N, d), n_ref, n_seq, n_slots = f["shape"], f["n_ref"], f["n_seq"], f["n_slots"]
    assert f["slot_stride"] == B * n_seq * d
    h0 = _rand(g, B, N, d, scale=2.0)
    slots = torch.randn(n_slots, B, n_seq, d, device="cuda", generator=g) * 0.5
    Rs, R = _flat(slots)
    outside = torch.ones(N, dtype=torch.bool, device="cuda")
    outside[n_ref:n_ref + n_seq] = False
    for coef, dead in _forecast_patterns(n_slots):
        what = f"step_cache_apply_forecast, coefficients {coef}" + ("" if dead is None else f", slot {dead} NaN")
        if dead is not None:
            R[dead].fill_(math.nan)
        Hs, h = _flat(h0)
        c = torch.tensor(coef + [math.nan] * (3 - n_slots), device="cuda")
        ops.step_cache_apply_forecast(h, R, c, n_ref)
        torch.cuda.synchronize()
        Hs.check(what), Rs.check(what)
        want = apply_forecast_ref(h0, slots, coef, n_ref)
        _exact(h, want, what)
        _exact(h[:, outside], h0[:, outside], what + ": ref and pose rows")
        if coef.count(1.0) == 1 and coef.count(0.0) == n_slots - 1:
            s = coef.index(1.0)
            plain = h0.clone()
            ops.step_cache_apply(plain, slots[s].contiguous(), n_ref)
            _exact(h, plain, what + ": step_cache_apply")
        if dead is not None:
            R[dead].copy_(slots[dead])
        _exact(R, slots, what + ": the slots (only read)")
        del Hs, h
    return f"exact for {len(_forecast_patterns(n_slots))} coefficient patterns over {n_slots} slots", 0.0


def check_unipc_step_(ops, f, g):
    """Bit for bit step_ref at the recorded coefficients, scale and sigma: x, x_last and the written slot; every slot with
    zero coefficients holds NaN-patterned sentinels (not read, and kept bit for bit unless written), and so does x_last
    when the corrector is off."""
    shape, n_slots, write, correct, coef = f["shape"], f["n_slots"], f["write_slot"], f["correct"], list(f["coef"])
    n = math.prod(shape)
    assert f["slot_stride"] == n
    x0 = torch.randn(*shape, device="cuda", generator=g)
    xl0 = torch.randn(*shape, device="cuda", generator=g) if correct else unipc_sentinel(1, n).view(shape).clone()
    v = (torch.randn(2, *shape[1:], device="cuda", generator=g) * 2.0).to(BF)
    before = unipc_sentinel(n_slots, n).clone()
    live = [s for s in range(n_slots) if coef[1 + s] != 0.0 or coef[6 + s] != 0.0]
    for s in live:
        before[s] = torch.randn(n, device="cuda", generator=g)
    z, y, m = step_ref(x0, xl0, v, before, f["scale"], f["sigma"], coef, correct)
    (X, x), (XL, xl), (V, vv), (S, slots) = _flat(x0), _flat(xl0), _flat(v), _flat(before)
    ops.unipc_step_(x, xl, vv, slots, write, f["scale"], f["sigma"], coef, correct)
    torch.cuda.synchronize()
    for s in (X, XL, V, S):
        s.check("unipc_step_")
    _exact(x.view(-1), z, "unipc_step_: x")
    _exact(xl.view(-1), y, "unipc_step_: x_last")
    _exact(slots[write], m, f"unipc_step_: slot {write}")
    for s in range(n_slots):
        if s != write:
            _exact(slots[s], before[s], f"unipc_step_: slot {s} (not written)")
    return f"exact; live slots {live}, write slot {write}, corrector {'on' if correct else 'off'}", 0.0


# ---------------------------------------------------------------- small kernels
def check_adaln_modulation(ops, f, g):
    B, n = f["shape"]
    emb, param = _rand(g, B, n), _rand(g, n, scale=0.3)
    c = assert_close_bf16(ops.adaln_modulation(emb, param), emb.float() + param.float(), "adaln_modulation")
    return _report(c), c.worst_ratio


def check_silu(ops, f, g):
    x = _rand(g, *f["shape"], scale=3.0)
    c = assert_close_bf16(ops.silu(x), F.silu(x.float()), "silu")
    return _report(c), c.worst_ratio


def check_timestep_embedding(ops, f, g):
    """At the sampler's real c_noise = 1000 sigma (50 steps, shift 5: up to 1000), fed in groups of the recorded batch."""
    from oracle import dit_oracle as O
    from scail_b200 import sampler
    B = f["B"]
    c_noise = sampler.make_flow_timesteps(50, 5.0)[:-1].cuda() * 1000.0
    worst, rl = 0.0, 0.0
    for i in range(0, len(c_noise) - B + 1, B):
        t = c_noise[i:i + B].contiguous()
        c = assert_close_bf16(ops.timestep_embedding(t, f["dim"]), O.timestep_embedding(t, f["dim"]), f"c_noise {t.tolist()}")
        worst, rl = max(worst, c.worst_ratio), max(rl, c.rel_l2)
    return f"rel-L2 <= {rl:.2e}, worst |d|/bound {worst:.2f} over c_noise 1000 .. {float(c_noise[-1]):.1f}", worst


def check_cast_bf16(ops, f, g):
    x = torch.randn(*f["shape"], device="cuda", generator=g) * 3
    return _exact(ops.cast_bf16(x), x.to(BF), "cast_bf16"), 0.0


def check_cfg_euler_(ops, f, g):
    shape, s, ds = f["shape"], f["scale"], f["dsigma"]
    x = torch.randn(*shape, device="cuda", generator=g)
    v = _rand(g, 2, *shape[1:])
    u, c = v[0:1].double(), v[1:2].double()
    want = x.double() + ds * (u + s * (c - u))
    got = ops.cfg_euler_(x.clone(), v, s, ds)
    # each fp32 operation rounds its own result once: 2^-24 of |x|, |ds u| and |ds s (c - u)| (before u cancels against
    # s (c - u)), a few times over, with or without FMA contraction
    bound = 2.0 ** -22 * (x.double().abs() + abs(ds) * (u.abs() + abs(s) * (c - u).abs()))
    ratio = float(((got.double() - want).abs() / bound.clamp_min(1e-300)).max())
    assert ratio <= 1, f"cfg_euler_: |d| / bound {ratio:.3g}"
    return f"worst |d|/bound {ratio:.2f}", ratio


def _patches(v):
    """O.patch_embed's gather: [b, t, c, h, w] -> [b, t * h/2 * w/2, c * 4]."""
    b, t, c, h, w = v.shape
    return v.reshape(b, t, c, h // 2, 2, w // 2, 2).permute(0, 1, 3, 5, 2, 4, 6).reshape(b, t * (h // 2) * (w // 2), c * 4)


def check_patchify(ops, f, g):
    B, Br, Bp, T, H, W, C = (f[k] for k in ("B", "Br", "Bp", "T", "H", "W", "C"))
    x, ref, pose = _rand(g, B, T, C, H, W), _rand(g, Br, 1, C, H, W), _rand(g, Bp, T, C, H // 2, W // 2)
    a_main, a_pose = ops.patchify(x, ref, pose)
    mask = lambda t, val: torch.cat([t, torch.full((*t.shape[:2], 4, *t.shape[3:]), val, device="cuda", dtype=BF)], 2)
    full = lambda t: (mask(t, 1.0) if C == 16 else t).expand(B, *t.shape[1:2], 20, *t.shape[3:])
    xm = mask(x, 0.0) if C == 16 else x
    _exact(a_main, _patches(torch.cat([full(ref), xm], 1)), "patchify ref || noise")
    return _exact(a_pose, _patches(full(pose)), "patchify pose"), 0.0


def check_unpatchify(ops, f, g):
    from oracle import dit_oracle as O
    B, T, Hp, Wp = f["B"], f["T"], f["Hp"], f["Wp"]
    n = T * Hp * Wp
    lin = _rand(g, B * n, 64)
    return _exact(ops.unpatchify(lin, B, T, Hp, Wp), O.unpatchify(lin.view(B, n, 64), 0, n, T, Hp, Wp), "unpatchify"), 0.0


def check_step_cache_indicator(ops, f, g):
    (B, N, d), n_ref, n_seq = f["shape"], f["n_ref"], f["n_seq"]
    h0, h1, r_ref = step_cache_operands(B, N, d, seed=N)
    r_new, h1c, partials, out = step_cache_scratch(B, N, d, n_seq)
    ops.step_cache_indicator(h0, h1, r_ref, r_new, h1c, n_ref, partials, out)
    r, num, den = indicator_sums(h0, h1, r_ref)
    _exact(r_new, r, "indicator r")
    _exact(h1c, h1[:, n_ref:n_ref + n_seq], "indicator h1c")
    got = out.tolist()
    assert abs(got[0] - num) <= 1e-6 * num and abs(got[1] - den) <= 1e-6 * den, (got, num, den)  # as test_step_cache_gpu
    return f"exact r and h1c; sums within {max(abs(got[0] - num) / num, abs(got[1] - den) / den):.1e} of fp64", 0.0


def check_step_cache_update(ops, f, g):
    (B, N, d), n_ref, n_seq = f["shape"], f["n_ref"], f["n_seq"]
    h1c, h = _rand(g, B, n_seq, d), _rand(g, B, N, d, scale=4.0)
    R = torch.empty(B, n_seq, d, device="cuda", dtype=torch.float32)
    ops.step_cache_update(h, h1c, R, n_ref)
    return _exact(R, update_ref(h, h1c, n_ref), "step_cache_update"), 0.0


def check_step_cache_apply(ops, f, g):
    (B, N, d), n_ref, n_seq = f["shape"], f["n_ref"], f["n_seq"]
    h, R = _rand(g, B, N, d), torch.randn(B, n_seq, d, device="cuda", generator=g)
    want = apply_ref(h, R, n_ref)
    ops.step_cache_apply(h, R, n_ref)
    return _exact(h, want, "step_cache_apply (noise rows changed, ref and pose rows not)"), 0.0


CHECKS = {name: globals()["check_" + name] for name in OPS}


def _describe(name, f):
    def fmt(v):
        if isinstance(v, tuple) and len(v) == 2 and hasattr(v[0], "seq_length"):  # (geometry, window)
            return f"({v[0].T}x{v[0].H}x{v[0].W}, window {v[1]})"
        return str(v).replace(" ", "")
    return name + " " + " ".join(f"{k}={fmt(v)}" for k, v in f.items())


def test_every_dit_launch_matches_fp32(launches):
    from scail_b200 import ops
    failures, worst = [], {}
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    print(f"\n{len(launches)} distinct DiT launches")
    for i, (name, f) in enumerate(launches):
        what = _describe(name, f)
        g = torch.Generator(device="cuda").manual_seed(2000 + i)
        try:
            result, ratio = CHECKS[name](ops, f, g)
            worst[name] = max(worst.get(name, 0.0), ratio)
            print(f"{what}: {result}")
        except AssertionError as e:
            print(f"FAIL {what}: {e}")
            failures.append(f"{what}: {e}")
        torch.cuda.empty_cache()
    print("worst |d|/bound per op (fp8 attention: worst block / (2 x chain's worst block + 1e-3); 0 = bit-exact): " +
          ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    print(f"{len(launches)} launches checked in {time.time() - t0:.0f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert not failures, f"{len(failures)} of {len(launches)} launches failed:\n" + "\n".join(failures)


def test_recorded_launches_cover_the_production_cases(launches):
    from scail_b200 import ops

    def has(name, **want):
        return any(n == name and all(v(f[k]) if callable(v) else f[k] == v for k, v in want.items()) for n, f in launches)

    Ns = {geo: (1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4) for geo, (t, h, w) in GEOMETRIES.items()}
    n_ref = {geo: (h // 2) * (w // 2) for geo, (t, h, w) in GEOMETRIES.items()}
    n_seq = {geo: t * (h // 2) * (w // 2) for geo, (t, h, w) in GEOMETRIES.items()}
    ld = lambda n: (lambda v: v[0] == n)
    grid = lambda geo: (GEOMETRIES[geo][0], GEOMETRIES[geo][1] // 2, GEOMETRIES[geo][2] // 2)
    window = lambda geo: (lambda t: t is not None and (t[0].T, t[0].H, t[0].W) == grid(geo) and t[1] == 2)
    gate_res = dict(epilogue=ops.EPI_BIAS_GATE_RES, rows_per_batch=lambda r: r % 128 != 0)
    cases = {
        "self-attention at B = 2, H = 40, L = 27904 / 42510 / 48832, Q/K/V slabs with ld 15360":
            all(has("attention", B=2, H=40, q_len=N, kv_len=N, q=ld(15360), k=ld(15360), v=ld(15360)) for N in Ns.values()),
        "cross-attention over 512 text keys, then 257 CLIP keys accumulated, at every geometry":
            all(has("attention", B=2, q_len=N, kv_len=512, accumulate=False) and
                has("attention", B=2, q_len=N, kv_len=257, accumulate=True) for N in Ns.values()),
        "bf16 and fp8 gate-residual GEMMs with rows_per_batch not a multiple of 128":
            has("gemm", **gate_res) and has("gemm_fp8", **gate_res),
        "final-layer ln_modulate with row_offset = n_ref at every geometry":
            all(has("ln_modulate", n_in=Ns[geo], row_offset=n_ref[geo], rows_out=n_seq[geo]) for geo in GEOMETRIES),
        "two-slab rmsnorm_rope with RoPE at every geometry":
            all(has("rmsnorm_rope", slabs=(0, 5120), rope=grid(geo) + (0, 0, 0), fp8=None) for geo in GEOMETRIES),
        "fp8 forms: GEMM, quantisers, LN, RMSNorm+RoPE and dense attention at every geometry":
            has("gemm_fp8") and has("quant_rows_fp8") and has("ln_modulate", fp8=True) and
            all(has("rmsnorm_rope", rope=grid(geo) + (0, 0, 0), fp8=lambda v: v is not None) and has("quant_vt_fp8", L=N) and
                has("attention_fp8", B=2, L=N, tiles=None) for geo, N in Ns.items()),
        "window-2 sparse maps, bf16 and fp8, at every geometry":
            all(has("attention_sparse", B=2, q_len=Ns[geo], tiles=window(geo)) and
                has("attention_fp8", B=2, L=Ns[geo], tiles=window(geo)) for geo in GEOMETRIES),
        "b = 1 forms at 512x896": has("attention", B=1, q_len=Ns[B1], kv_len=Ns[B1]) and
            has("gemm", M=Ns[B1], rows_per_batch=Ns[B1], epilogue=ops.EPI_BIAS_GATE_RES) and has("patchify", B=1),
        "step-cache indicator, update and apply at ragged N": all(
            has(op, shape=lambda s, N=Ns[geo]: s[:2] == (2, N)) for geo in CACHED
            for op in ("step_cache_indicator", "step_cache_update", "step_cache_apply")),
        "patchify with Br = Bp = 1 < B = 2": has("patchify", B=2, Br=1, Bp=1),
        "patch-embed GEMM writing a row range of hidden": has("gemm", K=80, out=lambda v: v[0] == 5120 and v[2]),
        "adaptive pooling (bf16 and fp8), selection and both per-(b, h) kernels at B = 2, H = 40, bf16 Q/K/V with ld 15360, "
        "at every geometry": all(
            has("tile_pool", B=2, H=40, L=N, fp8=False, x=ld(15360)) and has("tile_pool", B=2, H=40, L=N, fp8=True) and
            has("select_tiles", B=2, H=40, L=N, n_ref=n_ref[geo], mass=ADAPTIVE[0], max_tiles=ADAPTIVE[1]) and
            has("attention_sparse_bh", B=2, H=40, L=N, q=ld(15360), k=ld(15360), v=ld(15360)) and
            has("attention_fp8_sparse_bh", B=2, H=40, L=N) for geo, N in Ns.items()),
        "forecast update_slot and apply_forecast with 2 and 3 slots at ragged N": all(
            has(op, shape=lambda s, N=Ns[geo]: s[:2] == (2, N), n_slots=k) for geo in CACHED for k in (2, 3)
            for op in ("step_cache_update_slot", "step_cache_apply_forecast")),
        "UniPC(3) steps with and without the corrector on the 512x896 latent": all(
            has("unipc_step_", shape=(1, 21, 16, 64, 112), n_slots=3, correct=c) for c in (False, True)),
    }
    print("\n" + "\n".join(f"{'ok' if ok else 'MISSING'}: {what}" for what, ok in cases.items()))
    assert all(cases.values()), [what for what, ok in cases.items() if not ok]


# ---------------------------------------------------------------- the whole path vs the fp32 oracle
def test_full_width_block_at_480x832_cfg_batch_vs_oracle():
    """One 14B-width block plus the embeddings and the final layer at latent 21x60x104 (N = 42 510), b = 2: the CFG batch of
    two different text contexts, as sampler_step runs it.  Per branch, ours vs the fp32 oracle is bounded by the
    reference-style bf16 library chain's error (the test_scale_gpu rule) and by absolute ceilings."""
    import oracle.dit_oracle as O
    m = full_width_model(1, seed=5)
    x0, cond, uc = step_inputs(6, *GEOMETRIES["480x832"])
    x = torch.cat([x0, x0]).to(BF)
    ctx = torch.cat([uc["crossattn"], cond["crossattn"]])
    ref, pose, clip = cond["ref_concat"], cond["concat_smpl_render"], cond["image_clip_features"]
    ts = torch.full((2,), 500.0, device="cuda")
    cap = {}
    ad = m.mixins["adaln_layer"]
    orig = ad.layer_forward

    def lf(hid, mask, **kw):
        o = orig(hid, mask, **kw)
        cap["block"] = o.clone()
        return o

    ad.layer_forward = lf
    with torch.no_grad():
        got = m(x, timesteps=ts, context=ctx, ref_concat=ref, concat_smpl_render=pose, image_clip_features=clip).float()
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
            sd16 = {k: v.to(BF) for k, v in sd.items()}
            del sd
            lib, hid16 = O.dit_forward(sd16, x, ts, ctx, ref, pose, clip, 40, 1, return_hidden=True, dtype=BF)
            hid16 = hid16[1]
    finally:
        O.sdpa = old_sdpa
    for b, branch in enumerate(("uncond", "cond")):
        e_blk, e_out = rel(cap["block"][b], hid[b]), rel(got[b], want[b])
        l_blk, l_out = rel(hid16[b], hid[b]), rel(lib[b], want[b])
        print(f"480x832 block, b = 2, {branch} branch: ours vs fp32 oracle: block {e_blk:.3e} out {e_out:.3e} | "
              f"reference-style bf16 library chain vs fp32 oracle: block {l_blk:.3e} out {l_out:.3e}")
        assert e_blk < 6e-3 and e_out < 8e-3, (branch, e_blk, e_out)
        assert e_blk < 1.5 * l_blk + 1e-3 and e_out < 1.5 * l_out + 1e-3, (branch, e_blk, l_blk, e_out, l_out)
