"""The context-parallel DiT launches at 14B width against fp32, on one GPU, through an in-process stand-in rank.

Under context parallelism each rank launches kernels at shapes no one-GPU forward makes: self-attention of n_local = N / P
local queries against the P n_local gathered keys, K / V projections into one slot of the [B, P, n_local, d] gather buffer,
RMSNorm+RoPE on a row slice of the RoPE tables (token sharding) or on tables built with rope_H / W_shift (the pre-chunked
form, chunk_dim), and with ContextParallel.local_first attention_partial over key ranges that start and end inside a
128-key tile, then attention_merge.  At the real geometries n_local is ragged against the tile (512x896: 24 416 / 12 208 /
6 104 for P = 2 / 4 / 8; 480x832: 21 255; 512x512: 6 976 / 3 488), so every shard starts inside a TMA box.

LoopbackCP(P, rank) is a ContextParallel without a process group: the K / V all-gather and the token gather fill the other
ranks' slots with the rows a one-GPU forward of the same model on the same inputs produced there (its post-RMSNorm/RoPE K,
its V and its hidden state before the final layer), so one process runs exactly one rank's launches.

test_every_cp_launch_matches_fp32: the full-width two-block random model (test_dit_launch_shapes_gpu.full_width_model) runs
as ranks 0, 1 and P - 1 of: the token-sharded forward at 512x896 (P = 2, 4, 8), 480x832 (P = 2) and 512x512 (P = 4, 8),
b = 2 (the CFG batch on two branch streams) and b = 1 (a HybridParallel rank), with and without fp8 linears; local_first at
512x896 (P = 4, 8) and 480x832 (P = 2); and the pre-chunked form with chunk_dim 3 and 4 at 512x896 (P = 2, 4) and chunk_dim
4 at 480x832 (P = 2).  Every DiT entry point plus attention_partial and attention_merge is recorded, and every distinct
launch is re-run on fresh data inside sentinel buffers by the checks of test_dit_launch_shapes_gpu.py (RMSNorm+RoPE on the
recorded table slice or shift; attention at q_len != kv_len with planted keys at the first and last key of every shard) and
the two below:
  attention_partial: o32 against the fp64 softmax over the union of the ranges' keys to the bf16-attention bound, the state
    (m, l) against its fp64 restatement to a bound derived from the fp32 arithmetic (check_attention_partial); a key just
    past a range inside the range's last TMA box (for the remote partial: the local shard's first key) must have no effect,
    and the first key of the local range must carry its row.
  attention_merge: on the kernel's own partials, one bf16 rounding from the fp64 merge of those partials and within the
    attention bound of fp32 attention over all keys; on synthetic partials with equal maxima, |m_a - m_b| up to 40 either
    way, and one side's weight underflowing to 0.
test_whole_cp_path_matches_one_gpu: each emulated rank's block outputs and output rows against the one-GPU forward: bit for
bit in the token-sharded form (the same key order and key tiles, per-row GEMMs); where the key order or the softmax max
differs (local_first's two partials; chunk_dim, whose gathered keys are in rank order, a permutation of the one-GPU order)
within twice the bf16 rel-L2 bound, and the local_first block 0 at 480x832 also against the fp32 oracle block."""
import math
import time

import pytest
import torch

from kernel_check import assert_close_bf16, recording
from test_dit_launch_shapes_gpu import (ATT_ELEM, BF, CHECKS, GEOMETRIES, LOGIT_STD, OPS, Slab, _attention_ref, _describe,
                                        _fields, _no_tf32, _rand, _report, _view, full_width_model, rel, step_inputs)
from test_host_cpu import chunk_tokens

from scail_b200.parallel import ContextParallel

pytestmark = pytest.mark.gpu
_no_tf32 = _no_tf32  # autouse: TF32 off in every test of this module

CP_OPS = OPS + ("attention_partial", "attention_merge")
TOKEN = [("512x896", 2), ("512x896", 4), ("512x896", 8), ("480x832", 2), ("512x512", 4), ("512x512", 8)]
LOCAL_FIRST = [("512x896", 4), ("512x896", 8), ("480x832", 2)]
CHUNKED = [("512x896", 3, 2), ("512x896", 3, 4), ("512x896", 4, 2), ("512x896", 4, 4), ("480x832", 4, 2)]
ORACLE = ("480x832", 2, 1)  # (geometry, P, rank) of the local_first block compared with the fp32 oracle
BF16_CHAINS = 8e-3  # rel-L2 of two bf16 chains that each stay within kernel_check's 4e-3 of the same fp32 function


def ranks(P):
    return sorted({0, 1, P - 1})


def seq_len(t, h, w):
    return (1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4)


# ---------------------------------------------------------------- the stand-in rank
class _Done:
    def wait(self):
        pass


class LoopbackCP(ContextParallel):
    """Rank `rank` of a P-way ContextParallel in one process, without a process group.  ref: the one-GPU forward's rows
    (Reference); index[p]: the one-GPU token rows of rank p's local sequence.  With b = 2 the branches run on
    branch_streams, so the current stream tells which batch row a gather is for."""

    def __init__(self, P, rank, ref, index):
        self.size, self.rank, self._handle = P, rank, None
        self._kv, self._q, self._streams = {}, {}, {}
        self.local_first = False
        self.ref, self.index, self._calls = ref, index, {}

    def _branch(self):
        cur = torch.cuda.current_stream().cuda_stream
        for ss in self._streams.values():
            for i, s in enumerate(ss):
                if s.cuda_stream == cur:
                    return i
        raise AssertionError("a gather outside the branch streams")

    def gather_kv(self, kvbuf, async_op=True):
        """Every slot but [0, rank] gets the K (a branch's first gather of a layer) or V (its second) rows of rank p."""
        i = self._branch()
        c = self._calls.get(i, 0)
        self._calls[i] = c + 1
        src = self.ref.kv[c // 2][c % 2]
        assert kvbuf.shape[0] == 1 and kvbuf.shape[1] == self.size
        for p in range(self.size):
            if p != self.rank:
                kvbuf[0, p].copy_(src[i, self.index[p]])
        return [_Done()]

    def gather_tokens(self, local, n_total):
        out = torch.empty(local.shape[0], n_total, local.shape[2], device=local.device, dtype=local.dtype)
        for p in range(self.size):
            out[:, self.index[p]] = local if p == self.rank else self.ref.final_hidden[:, self.index[p]]
        return out


# ---------------------------------------------------------------- one-GPU reference and emulated ranks
class Reference:
    """The one-GPU forward's post-RMSNorm/RoPE K and V per layer ([b, N, d] each), block outputs, hidden state before the
    final layer and output."""


def _inputs(geo, b, seed):
    t, h, w = GEOMETRIES[geo]
    x0, cond, uc = step_inputs(seed, t, h, w)
    x = torch.cat([x0, x0]).to(BF) if b == 2 else x0.to(BF)
    ctx = torch.cat([uc["crossattn"], cond["crossattn"]]) if b == 2 else cond["crossattn"]
    return dict(x=x, timesteps=torch.full((b,), 500.0, device="cuda"), context=ctx, ref_concat=cond["ref_concat"],
                concat_smpl_render=cond["concat_smpl_render"], image_clip_features=cond["image_clip_features"])


def _capture_blocks(ad, into):
    orig = ad.layer_forward

    def lf(hid, mask, **kw):
        o = orig(hid, mask, **kw)
        into.append(o.clone())
        return o
    ad.layer_forward = lf
    return lambda: delattr(ad, "layer_forward")


def reference(m, inp):
    from scail_b200 import ops
    ad, fl = m.mixins["adaln_layer"], m.mixins["final_layer"]
    r = Reference()
    r.kv, r.blocks = [], []
    d = m.hidden_size
    orig_rr, orig_ff = ops.rmsnorm_rope, fl.final_forward

    def rr(buf, rows_per_batch, D, slabs, *a, **k):
        out = orig_rr(buf, rows_per_batch, D, slabs, *a, **k)
        if len(slabs) == 2:  # the self-attention Q | K normalisation of the fused QKV buffer
            B = buf.shape[0] // rows_per_batch
            r.kv.append((buf[:, d:2 * d].clone().view(B, rows_per_batch, d), buf[:, 2 * d:].clone().view(B, rows_per_batch, d)))
        return out

    def ff(hidden, **kw):
        r.final_hidden = hidden.clone()
        return orig_ff(hidden, **kw)
    ops.rmsnorm_rope, fl.final_forward = rr, ff
    restore = _capture_blocks(ad, r.blocks)
    try:
        r.out = m(**inp)
    finally:
        ops.rmsnorm_rope = orig_rr
        del fl.final_forward
        restore()
    torch.cuda.synchronize()
    assert len(r.kv) == len(r.blocks) == m.num_layers
    return r


def run_rank(m, inp, ref, P, rank, local_first=False, chunk_dim=None):
    """The forward of rank `rank` -> (output, [block output per (layer, branch)], index of every rank's token rows)."""
    ad = m.mixins["adaln_layer"]
    t, h, w = inp["x"].shape[1], inp["x"].shape[3], inp["x"].shape[4]
    N = seq_len(t, h, w)
    if chunk_dim is None:
        n = N // P
        index = [torch.arange(p * n, (p + 1) * n, device="cuda") for p in range(P)]
        kw = inp
    else:
        index = [chunk_tokens(t, h // 2, w // 2, chunk_dim, P, p).cuda() for p in range(P)]
        part = lambda a: a.chunk(P, chunk_dim)[rank].contiguous()
        kw = dict(inp, x=part(inp["x"]), ref_concat=part(inp["ref_concat"]), concat_smpl_render=part(inp["concat_smpl_render"]),
                  chunk_dim=chunk_dim)
    cp = LoopbackCP(P, rank, ref, index)
    cp.local_first = local_first
    ad.cp = cp
    blocks = []
    restore = _capture_blocks(ad, blocks)
    try:
        out = m(**kw)
        torch.cuda.synchronize()
    finally:
        restore()
        ad.cp = None
    return out, blocks, index


def compare_rank(out, blocks, ref, P, rank, index, chunk_dim=None):
    """Block outputs and output rows of this rank against the one-GPU forward -> {what: (bit-identical, rel-L2)}."""
    b = ref.out.shape[0]
    res = {}
    for j, got in enumerate(blocks):  # in (layer, branch) order
        l, i = divmod(j, b)
        want = ref.blocks[l][i:i + 1, index[rank]]
        res[f"block {l}, branch {i}"] = (torch.equal(got, want), rel(got, want))
    want = ref.out if chunk_dim is None else ref.out.chunk(P, chunk_dim)[rank]
    res["output"] = (torch.equal(out, want), rel(out, want))
    return res


# ---------------------------------------------------------------- recording
def _cp_fields(name, a):
    if name == "attention_partial":
        q_len = a["q_len"]
        assert a["kv_batch_rows"] is not None
        return dict(B=a["B"], H=a["H"], q_len=q_len, ranges=tuple((int(o), int(n)) for o, n in a["ranges"]),
                    q_rows=q_len if a["q_batch_rows"] is None else a["q_batch_rows"], kv_rows=a["kv_batch_rows"],
                    q=_view(a["q"]), k=_view(a["k"]), v=_view(a["v"]), o32=_view(a["o32"]), q_total=a["q"].shape[0],
                    kv_total=a["k"].shape[0], scale=float(a["scale"] or 1.0 / math.sqrt(128))), 1
    if name == "attention_merge":
        return dict(rows=a["out"].shape[0], H=a["H"], o32=_view(a["o32_a"]), out=_view(a["out"])), 1
    return _fields(name, a)


@pytest.fixture(scope="module")
def cp_runs():
    """(launches [(op, key)] in first-call order, whole-path results [(case, {what: (bit-identical, rel-L2)})], the oracle
    comparison of ORACLE's block 0)."""
    from scail_b200 import dit, ops
    m = full_width_model(2)
    ad = m.mixins["adaln_layer"]
    seen_all, whole, oracle = {}, [], None
    with torch.no_grad():
        for gi, geo in enumerate(GEOMETRIES):
            for b, fp8 in ((2, False), (1, False), (2, True), (1, True)):
                jobs = [(P, r, False, None) for g, P in TOKEN if g == geo for r in ranks(P)]
                if (b, fp8) == (2, False):
                    jobs += [(P, r, True, None) for g, P in LOCAL_FIRST if g == geo for r in ranks(P)]
                    jobs += [(P, r, False, cd) for g, cd, P in CHUNKED if g == geo for r in ranks(P)]
                if not jobs:
                    continue
                ad.fp8_linear = fp8
                inp = _inputs(geo, b, 40 + gi)
                ref = reference(m, inp)
                for P, r, lf, cd in jobs:
                    with recording(ops, CP_OPS, _cp_fields) as seen:
                        out, blocks, index = run_rank(m, inp, ref, P, r, lf, cd)
                    for k in seen:
                        seen_all.setdefault(k, None)
                    case = (f"{geo} P={P} rank {r} b={b}" + (" fp8 linears" if fp8 else "") + (" local_first" if lf else "") +
                            (f" chunk_dim={cd}" if cd else ""))
                    whole.append((case, not lf and cd is None, compare_rank(out, blocks, ref, P, r, index, cd)))
                    if (geo, P, r) == ORACLE and lf:
                        oracle = _oracle_block0(m, inp, blocks, index[r])
                    del out, blocks
                ad.fp8_linear = False
                del ref, inp
                torch.cuda.synchronize()
                dit._WS.bufs.clear()
                torch.cuda.empty_cache()
    del m, ad
    dit._WS.bufs.clear()
    torch.cuda.empty_cache()
    return [(name, dict(k)) for (name, k) in seen_all], whole, oracle


def _oracle_block0(m, inp, blocks, rows):
    """rel-L2 per branch of this rank's block-0 rows against the fp32 oracle (embeddings + block 0 on the whole sequence)."""
    import oracle.dit_oracle as O
    from test_scale_gpu import sdpa_fp32_chunked
    sd = {k: v.float() for k, v in m.state_dict().items()}
    old = O.sdpa
    O.sdpa = lambda q, k, v: sdpa_fp32_chunked(q, k, v) if q.dtype == torch.float32 else old(q, k, v)
    try:
        with torch.device("cuda"):
            _, hid = O.dit_forward(sd, inp["x"].float(), inp["timesteps"], inp["context"].float(), inp["ref_concat"].float(),
                                   inp["concat_smpl_render"].float(), inp["image_clip_features"].float(), 40, 1,
                                   return_hidden=True)
    finally:
        O.sdpa = old
    del sd
    want = hid[1][:, rows]
    del hid
    res = [rel(blocks[i], want[i:i + 1]) for i in range(want.shape[0])]  # blocks[i]: layer 0, branch i
    torch.cuda.empty_cache()
    return res


# ---------------------------------------------------------------- attention_partial and attention_merge
_LOG2E = 1.4426950408889634


def _partial_ref64(q, k, v, H, scale):
    """fp64 softmax(scale q k^T) v of one batch over all rows of k, v ([rows, H*128]) -> (o, m, l, A): m the row max of
    scale log2(e) q k in log2 units, l = sum 2^(scale log2(e) q k - m), A = max over keys of sum_d |q_d k_d| ([rows, H])."""
    n = q.shape[0]
    c = scale * _LOG2E
    o = torch.empty(n, H * 128, device="cuda", dtype=torch.float64)
    m, l, A = (torch.empty(n, H, device="cuda", dtype=torch.float64) for _ in range(3))
    chunk = max(128, (2 ** 27 // k.shape[0]) // 128 * 128)
    for h in range(H):
        cols = slice(h * 128, h * 128 + 128)
        kh, vh = k[:, cols].double(), v[:, cols].double()
        ka = kh.abs().T.contiguous()
        kt = kh.T.contiguous()
        for i in range(0, n, chunk):
            qh = q[i:i + chunk, cols].double()
            s = (qh @ kt) * c
            mm = s.amax(-1)
            p = torch.exp2(s.sub_(mm[:, None]))
            ll = p.sum(-1)
            o[i:i + chunk, cols] = (p @ vh) / ll[:, None]
            m[i:i + chunk, h], l[i:i + chunk, h] = mm, ll
            A[i:i + chunk, h] = (qh.abs() @ ka).amax(-1)
            del s, p
    return o, m, l, A


def _state_bounds(m, A, n_tiles, scale):
    """Bounds on |m^ - m| and |l^ - l| / l of the kernel's fp32 state against the fp64 restatement (u = 2^-24):
      logits: the tensor core adds 128 exact bf16 products in fp32, at most one ulp (2u relative) per addition whether it
        rounds or truncates: |s^ - s| <= 128 * 2u * sum|q_d k_d| = 2^-16 A.
      c = scale log2(e) in fp32: fl(fl(scale) * fl(log2 e)), three roundings: |c^ - c| <= 3u c.
      m^ = fl(max(s^) c^): |m^ - m| <= c 2^-16 A + 5u (|m| + c A)  (the 3u of c^, the product's rounding, and margin).
      l^ = sum of ex2.approx(fma(s^, c^, -m^)) in fp32: each argument is off by at most c 2^-16 A + 3u c A (s^, c^) plus
        |m^ - m| plus one rounding of the fma (u (c A + |m|)); a relative change of 2^e in a term is ln 2 e; ex2.approx adds
        2^-21 relative (ftz: results below 2^-126 flush, which moves l >= 1 by less than 2^-100).  Each thread adds its 32
        keys of every 128-key tile sequentially and a quad reduction adds 2 more: (32 n_tiles + 2) additions, each at most
        u of the (positive) partial sum.  At most n_tiles rescales l *= 2^(m_old - m_new) (ex2.approx and one rounding).
    -> (dm [rows, H], dl_rel [rows, H])."""
    u = 2.0 ** -24
    c = scale * _LOG2E
    dm = c * 2.0 ** -16 * A + 5 * u * (m.abs() + c * A)
    arg = c * 2.0 ** -16 * A + 3 * u * c * A + dm + u * (c * A + m.abs())
    dl = math.log(2) * arg * 1.01 + 2.0 ** -21 + (32 * n_tiles + 2) * u * 1.01 + n_tiles * (2.0 ** -21 + u)
    return dm, dl


def _in_ranges(key, ranges):
    return any(o <= key < o + n for o, n in ranges)


def check_attention_partial(ops, f, g):
    B, H, q_len, ranges, kv_rows, scale = f["B"], f["H"], f["q_len"], f["ranges"], f["kv_rows"], f["scale"]
    assert f["q_rows"] == q_len and f["q_total"] == B * q_len and f["kv_total"] == B * kv_rows
    s = LOGIT_STD ** 0.5
    q, k, v = _rand(g, B * q_len, H * 128, scale=s), _rand(g, B * kv_rows, H * 128, scale=s), _rand(g, B * kv_rows, H * 128)
    # batch 0: the first and last key of every range carry a row (alpha 0.5: about 0.9 of its weight); the key just past a
    # range's end lies inside the range's last TMA box whenever the range ends mid-tile (for the remote partial's first
    # range: the local shard's first key) and must have no effect at alpha 1 (where it would take all of the weight)
    plants, masked = [], []
    for o, n in ranges:
        plants += [(o, 0.5), (o + n - 1, 0.5)]
        if o + n < kv_rows and not _in_ranges(o + n, ranges):
            masked.append(o + n)
            plants.append((o + n, 1.0))
    first = (ranges[0][0], 1.0)  # the first key of the first range at alpha 1 must carry its row
    plants.append(first)
    rows = []
    for j, (key, alpha) in enumerate(plants):
        row = 5 + 23 * j
        for h in (0, H - 1):
            cols = slice(h * 128, h * 128 + 128)
            q[row, cols] = (alpha * k[key, cols].float()).to(BF)
        rows.append((row, key, alpha))
    Q, K, V = Slab(q, f["q"]), Slab(k, f["k"]), Slab(v, f["v"])
    O = Slab(torch.zeros(B * q_len, H * 128, device="cuda"), f["o32"])
    S = Slab(torch.zeros(B * q_len, H * 2, device="cuda"), (H * 2, 0, True))
    ops.attention_partial(Q.v, K.v, V.v, O.v, S.v.view(B * q_len, H, 2), B, H, q_len, list(ranges), q_batch_rows=q_len,
                          kv_batch_rows=kv_rows, scale=scale)
    torch.cuda.synchronize()
    for sl in (Q, K, V, O, S):
        sl.check("attention_partial")
    sel = torch.cat([torch.arange(o, o + n) for o, n in ranges]).cuda()
    n_tiles = sum(-(-n // 128) for _, n in ranges)
    worst_o = worst_m = worst_l = 0.0
    reports = []
    for bi in range(B):
        qb = q[bi * q_len:(bi + 1) * q_len]
        kb, vb = k[bi * kv_rows:(bi + 1) * kv_rows][sel], v[bi * kv_rows:(bi + 1) * kv_rows][sel]
        o64, m64, l64, A = _partial_ref64(qb, kb, vb, H, scale)
        got = O.v[bi * q_len:(bi + 1) * q_len]
        c = assert_close_bf16(got, o64.float(), "attention_partial o32 vs the fp64 softmax over the ranges", **ATT_ELEM)
        worst_o = max(worst_o, c.worst_ratio)
        del o64
        st = S.v[bi * q_len:(bi + 1) * q_len].view(q_len, H, 2).double()
        dm, dl = _state_bounds(m64, A, n_tiles, scale)
        rm = float(((st[..., 0] - m64).abs() / dm).max())
        rl = float(((st[..., 1] - l64).abs() / (dl * l64)).max())
        assert rm <= 1, f"attention_partial: m off its fp64 restatement by {rm:.3g} x the bound"
        assert rl <= 1, f"attention_partial: l off its fp64 restatement by {rl:.3g} x the bound"
        worst_m, worst_l = max(worst_m, rm), max(worst_l, rl)
        if bi == 0:
            reports.append(f"max |dm| {float((st[..., 0] - m64).abs().max()):.2e} (bound {float(dm.max()):.2e}), max |dl|/l "
                           f"{float(((st[..., 1] - l64).abs() / l64).max()):.2e} (bound {float(dl.max()):.2e})")
        del m64, l64, A, dm, st
    row, key, _ = rows[-1]
    for h in (0, H - 1):  # the first key of the range carries its row: the output is that key's V, to a few bf16 roundings
        cols = slice(h * 128, h * 128 + 128)
        e = rel(O.v[row, cols], v[key, cols])
        assert e < 2e-2, f"attention_partial: row {row}, head {h} planted on key {key} (range start): rel-L2 vs V {e:.3e}"
    return (_report(c) + f"; state: {reports[0]}, |dm|/bound {worst_m:.2f}, |dl|/bound {worst_l:.2f}; {len(plants)} planted "
            f"keys, {len(masked)} past a range end"), max(worst_o, worst_m, worst_l)


def _merge64(oa, sa, ob, sb):
    """fp64 merge of two normalised partials with states (m, l) [rows, H, 2] -> [rows, H * 128]."""
    rows, H = sa.shape[:2]
    sa, sb = sa.double(), sb.double()
    m = torch.maximum(sa[..., 0], sb[..., 0])
    wa, wb = sa[..., 1] * torch.exp2(sa[..., 0] - m), sb[..., 1] * torch.exp2(sb[..., 0] - m)
    ca, cb = (wa / (wa + wb))[..., None], (wb / (wa + wb))[..., None]
    return (ca * oa.double().view(rows, H, 128) + cb * ob.double().view(rows, H, 128)).view(rows, H * 128)


def _merge(ops, f, oa, sa, ob, sb):
    """attention_merge at the recorded views, every operand inside sentinels -> the output view."""
    rows, H = f["rows"], f["H"]
    A, B_ = Slab(oa, f["o32"]), Slab(ob, f["o32"])
    SA, SB = Slab(sa.view(rows, 2 * H), (2 * H, 0, True)), Slab(sb.view(rows, 2 * H), (2 * H, 0, True))
    out = Slab(torch.zeros(rows, H * 128, device="cuda", dtype=BF), f["out"])
    ops.attention_merge(A.v, SA.v.view(rows, H, 2), B_.v, SB.v.view(rows, H, 2), out.v, H)
    torch.cuda.synchronize()
    for sl in (A, B_, SA, SB, out):
        sl.check("attention_merge")
    return out.v


def check_attention_merge(ops, f, g):
    rows, H = f["rows"], f["H"]
    # 1. on the kernel's own partials: rows local queries against a key set split as rank 1 of 3 splits it (a local range
    # that starts and ends mid-tile, the rest in two remote ranges)
    n = rows // 3
    kv = rows + 717
    local, remote = [(333, n)], [(0, 333), (333 + n, kv - 333 - n)]
    s = LOGIT_STD ** 0.5
    q, k, v = _rand(g, rows, H * 128, scale=s), _rand(g, kv, H * 128, scale=s), _rand(g, kv, H * 128)
    parts = []
    for ranges in (local, remote):
        o = torch.empty(rows, H * 128, device="cuda")
        st = torch.empty(rows, H, 2, device="cuda")
        ops.attention_partial(q, k, v, o, st, 1, H, rows, ranges, kv_batch_rows=kv)
        parts += [o, st]
    got = _merge(ops, f, *parts)
    c1 = assert_close_bf16(got, _merge64(*parts).float(), "attention_merge vs the fp64 merge of the kernel's partials")
    want = _attention_ref(q, k, v, 1, H, rows, kv, 1.0 / math.sqrt(128))
    c2 = assert_close_bf16(got, want, "attention_merge vs fp32 attention over all keys", **ATT_ELEM)
    del q, k, v, parts, want
    # 2. synthetic partials: m_b - m_a cycles through 0, small and large gaps either way, and +-160 (the smaller side's
    # weight 2^-160 underflows to 0 in fp32)
    gaps = torch.tensor([0.0, 0.0, 0.5, -0.5, 3.0, -3.0, 12.25, -12.25, 25.0, -25.0, 40.0, -40.0, 160.0, -160.0], device="cuda")
    items = rows * H
    ma = torch.rand(items, device="cuda", generator=g) * 45 - 5
    mb = ma + gaps[torch.arange(items, device="cuda") % len(gaps)]
    la = 1 + torch.rand(items, device="cuda", generator=g) * 3000
    lb = 1 + torch.rand(items, device="cuda", generator=g) * 3000
    sa, sb = torch.stack([ma, la], -1).view(rows, H, 2), torch.stack([mb, lb], -1).view(rows, H, 2)
    oa, ob = torch.randn(rows, H * 128, device="cuda", generator=g), torch.randn(rows, H * 128, device="cuda", generator=g)
    got = _merge(ops, f, oa, sa, ob, sb)
    c3 = assert_close_bf16(got, _merge64(oa, sa, ob, sb).float(), "attention_merge on synthetic partials")
    under = int((gaps[torch.arange(items, device="cuda") % len(gaps)].abs() == 160).sum())
    return (f"own partials: {_report(c1)} (one rounding); vs fp32 over all keys {_report(c2)}; synthetic: {_report(c3)}, "
            f"{under} (row, head) items with an underflowing side"), max(c1.worst_ratio, c2.worst_ratio,
                                                                                      c3.worst_ratio)


CP_CHECKS = dict(CHECKS, attention_partial=check_attention_partial, attention_merge=check_attention_merge)


# ---------------------------------------------------------------- tests
def test_every_cp_launch_matches_fp32(cp_runs):
    from scail_b200 import ops
    launches = cp_runs[0]
    failures, worst = [], {}
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    print(f"\n{len(launches)} distinct context-parallel DiT launches")
    for i, (name, f) in enumerate(launches):
        what = _describe(name, f)
        g = torch.Generator(device="cuda").manual_seed(3000 + i)
        try:
            result, ratio = CP_CHECKS[name](ops, f, g)
            worst[name] = max(worst.get(name, 0.0), ratio)
            print(f"{what}: {result}")
        except AssertionError as e:
            print(f"FAIL {what}: {e}")
            failures.append(f"{what}: {e}")
        torch.cuda.empty_cache()
    print("worst |d|/bound per op (0 = bit-exact): " + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    print(f"{len(launches)} launches checked in {time.time() - t0:.0f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert not failures, f"{len(failures)} of {len(launches)} launches failed:\n" + "\n".join(failures)


def test_recorded_cp_launches_cover_the_cases(cp_runs):
    launches = cp_runs[0]

    def has(name, **want):
        return any(n == name and all(v(f[k]) if callable(v) else f[k] == v for k, v in want.items()) for n, f in launches)

    Ns = {geo: seq_len(*GEOMETRIES[geo]) for geo in GEOMETRIES}
    grid = lambda geo: (GEOMETRIES[geo][0], GEOMETRIES[geo][1] // 2, GEOMETRIES[geo][2] // 2)
    pairs = sorted(set(TOKEN) | {(g, P) for g, _, P in CHUNKED})
    cases = {
        "self-attention of n_local queries against P n_local keys at every (geometry, P)":
            all(has("attention", B=1, H=40, q_len=Ns[g] // P, kv_len=Ns[g]) for g, P in pairs),
        "a partial whose range starts mid-tile": has("attention_partial", ranges=lambda r: any(o % 128 for o, _ in r)),
        "a two-range partial": has("attention_partial", ranges=lambda r: len(r) == 2),
        "a merge": has("attention_merge"),
        "every emulated rank's slice of the RoPE tables (token sharding)":
            all(has("rmsnorm_rope", rope=grid(g) + (0, 0, r * (Ns[g] // P))) for g, P in TOKEN for r in ranks(P)),
        "shifted tables on H and on W (chunk_dim 3 and 4)":
            has("rmsnorm_rope", rope=lambda t: t is not None and t[3] > 0 and t[5] == 0) and
            has("rmsnorm_rope", rope=lambda t: t is not None and t[4] > 0 and t[5] == 0),
        "fp8 projections on h_scale row slices": has("gemm_fp8", M=lambda M: any(M == Ns[g] // P for g, P in TOKEN)),
    }
    print("\n" + "\n".join(f"{'ok' if ok else 'MISSING'}: {what}" for what, ok in cases.items()))
    assert all(cases.values()), [what for what, ok in cases.items() if not ok]


def test_whole_cp_path_matches_one_gpu(cp_runs):
    """Token-sharded with local_first off: bit for bit (per row the same key order, key tiles and GEMM arithmetic as one GPU,
    measured bit-identical at every case here).  local_first and chunk_dim change which keys share a tile and the row max P
    is rounded against: P enters PV as bf16 relative to the running max, so it rounds differently, and under the nearly
    uniform softmax of random weights that moves the attention output by ~2^-9 of itself (measured: 2.3e-3 after block 0,
    3.1e-3 after block 1, up to 4.1e-3 at the output).  Both forwards are bf16 chains whose every launch is within
    kernel_check's rel-L2 bound (4e-3) of the same fp32 function, so their difference is bounded by twice that.  The
    local_first block 0 at ORACLE is also within the fp32-oracle bound of test_full_width_block_at_480x832_cfg_batch_vs_oracle
    (6e-3) on this rank's rows."""
    _, whole, oracle = cp_runs
    bad = []
    for case, exact, res in whole:
        line = ", ".join(f"{k} {'exact' if e else f'{r:.2e}'}" for k, (e, r) in res.items())
        print(f"{case}: {line}")
        for k, (e, r) in res.items():
            if (exact and not e) or (not exact and r > BF16_CHAINS):
                bad.append(f"{case}: {k}: {'not bit-identical, rel-L2 ' if exact else 'rel-L2 '}{r:.3e}")
    assert oracle is not None
    print(f"{ORACLE} local_first block 0 vs the fp32 oracle, per branch: " + ", ".join(f"{e:.3e}" for e in oracle))
    bad += [f"oracle block 0, branch {i}: {e:.3e} >= 6e-3" for i, e in enumerate(oracle) if e >= 6e-3]
    assert not bad, "\n".join(bad)


def test_cp_still_refuses_fp8_attention_windows_and_adaptive_maps():
    from scail_b200 import sparse
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    m = DiffusionTransformer(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=1, text_dim=64,
                             time_embed_dim=256).to(BF).cuda().eval()
    ad = m.mixins["adaln_layer"]
    t, h, w = 4, 16, 16
    inp = dict(x=torch.randn(2, t, 16, h, w, device="cuda").to(BF), timesteps=torch.full((2,), 500.0, device="cuda"),
               context=torch.randn(2, 32, 64, device="cuda").to(BF), ref_concat=torch.randn(1, 1, 16, h, w, device="cuda").to(BF),
               concat_smpl_render=torch.randn(1, t, 16, h // 2, w // 2, device="cuda").to(BF),
               image_clip_features=torch.randn(1, 257, 1280, device="cuda").to(BF))
    ad.cp = LoopbackCP(2, 0, None, None)
    for attr, val in (("fp8_attention", True), ("attention_window", 2), ("attention_adaptive", sparse.AdaptiveTiles(0.9, 40))):
        setattr(ad, attr, val)
        with torch.no_grad(), pytest.raises(NotImplementedError, match="context parallelism"):
            m(**inp)
        setattr(ad, attr, False if attr == "fp8_attention" else None)
