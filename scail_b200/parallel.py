"""Context parallelism for the DiT: tokens of the ref || noise || pose sequence are sharded contiguously over
the ranks of one process group; every per-token op (LN, GEMMs, RMSNorm/RoPE, cross-attention against the
replicated text/CLIP keys, MLP) is local, and self-attention needs ONE exchange per block: an NCCL all-gather
of the post-norm, post-RoPE K and V (SURVEY.md §8e).  Replaces the reference's Ulysses sequence parallelism
(sat/mpu/ulysses_attn_layer.py:41-110: 4 all_to_all_single per attention call, 12 per block) — numerically the
same softmax over the same key set, so parity is checked against the single-GPU path.

The all-gather is issued asynchronously (NCCL stream) right after the K/V projection so that the Q projection
and its RMSNorm+RoPE overlap the transfer.
"""
import ctypes
import os

import torch
import torch.distributed as dist

from . import ops


class _NativeWork:
    """Handle of collectives enqueued through libscail_b200's scail_cp_allgather: wait() makes the CURRENT stream wait (device
    side) for the group's communication stream, like torch.distributed's Work.wait() does for NCCL work."""

    def __init__(self, handle):
        self.handle = handle

    def wait(self):
        from . import _lib
        _lib.check(_lib.lib().scail_cp_wait(self.handle, torch.cuda.current_stream().cuda_stream), "scail_cp_wait")


class ContextParallel:
    def __init__(self, group=None, native=None):
        """native=True routes the K/V all-gather through the library's own NCCL communicator and communication stream
        (scail_cp_* in the C ABI: SURVEY 8b "collective"); False uses torch.distributed.all_gather_into_tensor.  Default: the
        SCAIL_CP_NATIVE environment variable (off unless set to 1)."""
        self.group = group if group is not None else dist.group.WORLD
        self.size = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self._handle = None
        if native is None:
            native = os.environ.get("SCAIL_CP_NATIVE", "0") == "1"
        if native and self.size > 1 and torch.cuda.is_available() and dist.get_backend(self.group) == "nccl":
            self._init_native()
        self._kv = {}
        self._q = {}
        self._streams = {}
        # Opt-in: attend to the local K/V shard first while the all-gathers are in flight, then to the remote shards, and merge
        # the two partials (scail_attention_partial / scail_attention_merge).  Two launches + fp32 partials + merge add work
        # that only pays off when the gather is exposed, and outputs are then no longer bit-identical to one GPU.  Off by
        # default; kept for larger CP degrees / slower links.
        self.local_first = False

    def _init_native(self):
        from . import _lib
        h = _lib.lib()
        uid = torch.zeros(128, dtype=torch.uint8)
        if self.rank == 0:
            buf = (ctypes.c_char * 128)()
            _lib.check(h.scail_cp_unique_id(ctypes.cast(buf, ctypes.c_void_p), None), "scail_cp_unique_id")
            uid = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        uid = uid.cuda()  # the id travels over the existing torch.distributed group (host-side plumbing)
        dist.broadcast(uid, src=dist.get_global_rank(self.group, 0), group=self.group)
        raw = bytes(uid.cpu().tolist())
        rc = h.scail_cp_init(ctypes.cast(ctypes.create_string_buffer(raw, 128), ctypes.c_void_p), self.rank, self.size, None)
        if rc < 0:
            _lib.check(rc, "scail_cp_init")
        self._handle = rc

    def branch_streams(self, n, device):
        key = (n, str(device))
        if key not in self._streams:
            self._streams[key] = [torch.cuda.Stream(device=device) for _ in range(n)]
        return self._streams[key]

    # ---- token sharding (kernel-free: also exercised on CPU/gloo by tests/test_parallel_cpu.py) ----
    def local_len(self, n_total):
        if n_total % self.size:
            raise ValueError(f"sequence length {n_total} is not divisible by the context-parallel size {self.size}")
        return n_total // self.size

    def shard_tokens(self, hidden):
        """[B, N, d] -> this rank's contiguous [B, N/P, d] chunk."""
        n = self.local_len(hidden.shape[1])
        return hidden[:, self.rank * n:(self.rank + 1) * n].contiguous()

    def gather_tokens(self, local, n_total):
        """[B, N/P, d] on every rank -> [B, N, d] on every rank."""
        B, n, d = local.shape
        buf = torch.empty(self.size * B, n, d, device=local.device, dtype=local.dtype)  # concatenated along dim 0
        dist.all_gather_into_tensor(buf, local.contiguous(), group=self.group)
        return buf.view(self.size, B, n, d).permute(1, 0, 2, 3).reshape(B, n_total, d)

    def rope_slice(self, cos, sin, n_local):
        s = slice(self.rank * n_local, (self.rank + 1) * n_local)
        return cos[s], sin[s]

    def kv_buffer(self, B, n_local, d, device, dtype=torch.bfloat16, width=None, tag="kv"):
        """[B, P, N/P, width] (default width 2d = K | V): batch-major so that, after the gather, batch b's keys/values are
        the contiguous [P*N/P, width] matrix the attention kernel addresses with kv_batch_rows = N."""
        width = 2 * d if width is None else width
        sid = torch.cuda.current_stream(device).cuda_stream if torch.device(device).type == "cuda" else 0
        key = (tag, B, n_local, width, str(device), dtype, sid)  # one buffer per stream (CFG branches run concurrently)
        if key not in self._kv:
            self._kv[key] = torch.empty(B, self.size, n_local, width, device=device, dtype=dtype)
        return self._kv[key]

    def gather_kv(self, kvbuf, async_op=True):
        """In-place all-gather per batch element: rank r's slot kvbuf[b, r] is sent, kvbuf[b] receives all."""
        B, P, n, w = kvbuf.shape
        if self._handle is not None:
            from . import _lib
            st = torch.cuda.current_stream(kvbuf.device).cuda_stream
            nbytes = n * w * kvbuf.element_size()
            for b in range(B):
                _lib.check(_lib.lib().scail_cp_allgather(self._handle, kvbuf[b, self.rank].data_ptr(), kvbuf[b].data_ptr(), nbytes,
                                                         st), "scail_cp_allgather")
            return [_NativeWork(self._handle)]
        works = []
        for b in range(B):
            works.append(dist.all_gather_into_tensor(kvbuf[b].view(P * n, w), kvbuf[b, self.rank], group=self.group,
                                                     async_op=async_op))
        return works

    # ---- the block's self-attention under CP (kernels) ----
    def self_attention(self, mixin, attn, h2, B, n_local, d, H, wq, wk, cos, sin, ctx, tables_local=False, h_scale=None):
        """tables_local: cos/sin already describe this rank's tokens (engine-style pre-chunked latents whose RoPE offsets
        come from rope_H/W_shift); otherwise they cover the full sequence and this rank's contiguous slice is taken.
        Keys/values are gathered in rank order either way (softmax is order-free).  h2 e4m3 with row scales h_scale
        (mixin.fp8_linear): the K, V and Q projections are fp8 GEMMs on row slices of the e4m3 QKV weight."""
        dev = h2.device
        P = self.size
        eps = mixin.layernorm_epsilon
        if tables_local:
            if cos.shape[0] != n_local:
                raise ValueError(f"pre-chunked context parallelism: RoPE tables have {cos.shape[0]} rows for {n_local} local tokens")
            cos_l, sin_l = cos, sin
        else:
            if cos.shape[0] != P * n_local:
                raise ValueError(f"context parallelism: RoPE tables have {cos.shape[0]} rows but P * n_local = {P} * {n_local}; "
                                 "tokens must be sharded with shard_tokens() (or pass chunk_dim for pre-chunked latents)")
            cos_l, sin_l = self.rope_slice(cos, sin, n_local)
        w, bias = attn.query_key_value.weight, attn.query_key_value.bias
        if h2.dtype == ops.FP8:
            w8, ws8 = mixin.fp8_weight(attn.query_key_value)

        def proj(rows, cols, out):  # out = h2[rows] @ w[cols]^T + bias[cols]; per-row scales slice with the rows
            if h2.dtype == ops.FP8:
                return ops.gemm_fp8(h2[rows], h_scale[rows], w8[cols], ws8[cols], bias[cols], out=out)
            return ops.gemm(h2[rows], w[cols], bias[cols], out=out)
        # K and V travel separately so that the K gather is already in flight during the V (and Q) projection and the V gather
        # during the Q projection: with one CFG branch per rank (HybridParallel) there is no second stream to hide it behind
        kbuf = self.kv_buffer(B, n_local, d, dev, width=d, tag="k")
        vbuf = self.kv_buffer(B, n_local, d, dev, width=d, tag="v")
        for b in range(B):  # K projection + RMSNorm/RoPE straight into this rank's slot of the gather buffer
            slot = kbuf[b, self.rank]
            proj(slice(b * n_local, (b + 1) * n_local), slice(d, 2 * d), slot)
            ops.rmsnorm_rope(slot, n_local, d, [(0, wk)], cos_l, sin_l, eps=eps)
        works = self.gather_kv(kbuf, async_op=True)
        for b in range(B):
            proj(slice(b * n_local, (b + 1) * n_local), slice(2 * d, 3 * d), vbuf[b, self.rank])
        works += self.gather_kv(vbuf, async_op=True)
        qkey = (B * n_local, d, str(dev), torch.cuda.current_stream(dev).cuda_stream)
        if qkey not in self._q:
            self._q[qkey] = torch.empty(B * n_local, d, device=dev, dtype=torch.bfloat16)
        q = self._q[qkey]
        proj(slice(None), slice(0, d), q)  # overlaps the all-gathers
        ops.rmsnorm_rope(q, n_local, d, [(0, wq)], cos_l, sin_l, eps=eps)
        k2, v2 = kbuf.view(B * P * n_local, d), vbuf.view(B * P * n_local, d)
        if not self.local_first:
            for wk_ in works:
                wk_.wait()
            ops.attention(q, k2, v2, ctx, B, H, n_local, P * n_local, q_batch_rows=n_local, kv_batch_rows=P * n_local)
            return ctx
        # Local shard first (SURVEY 8e: "attention over the local K/V shard starts immediately; remote shards consumed as
        # they arrive"): the partial over this rank's own keys runs while the all-gathers are in flight, the partial over all
        # other shards once they have landed; the two are merged with their softmax statistics (fp32 partials: the only
        # difference to one pass over all keys is fp32 summation order).
        o_a, st_a, o_b, st_b = self._partials(B * n_local, d, H, dev)
        r = self.rank
        ops.attention_partial(q, k2, v2, o_a, st_a, B, H, n_local, [(r * n_local, n_local)], q_batch_rows=n_local,
                              kv_batch_rows=P * n_local)
        for wk_ in works:
            wk_.wait()
        remote = [(o, l) for (o, l) in ((0, r * n_local), ((r + 1) * n_local, (P - 1 - r) * n_local)) if l > 0]
        ops.attention_partial(q, k2, v2, o_b, st_b, B, H, n_local, remote, q_batch_rows=n_local, kv_batch_rows=P * n_local)
        ops.attention_merge(o_a, st_a, o_b, st_b, ctx, H)
        return ctx

    def _partials(self, rows, d, H, dev):
        key = ("partials", rows, d, H, str(dev), torch.cuda.current_stream(dev).cuda_stream)
        if key not in self._q:
            self._q[key] = (torch.empty(rows, d, device=dev, dtype=torch.float32), torch.empty(rows, H, 2, device=dev, dtype=torch.float32),
                            torch.empty(rows, d, device=dev, dtype=torch.float32), torch.empty(rows, H, 2, device=dev, dtype=torch.float32))
        return self._q[key]


class HybridParallel:
    """CFG-parallel x context-parallel layout (SURVEY.md §8f rank 3).  The two classifier-free-guidance branches of a sampler
    step are independent forwards (guiders.py:47-57 only concatenates them on the batch axis), so with an even world size
    W = 2 * cp_size the ranks split into two halves: ranks [0, cp_size) run the UNCOND branch, ranks [cp_size, W) the COND
    branch, each half with context parallelism over its own cp_size ranks (b = 1 per rank: every GEMM / attention launch has
    twice the rows per rank of the pure-CP layout at the same W, and the K/V all-gather volume per rank halves).  The only
    cross-half traffic is one all-gather of the branch velocity (5.5 MB at 512p/81f) per step between partner ranks
    (i, i + cp_size), after which every rank applies the same CFG combine + Euler update to its replicated fp32 latent.
    W = 2 is pure CFG parallelism (no K/V collective at all)."""

    def __init__(self):
        world, rank = dist.get_world_size(), dist.get_rank()
        if world % 2:
            raise ValueError(f"HybridParallel needs an even world size, got {world}")
        self.world, self.rank = world, rank
        self.cp_size = world // 2
        self.branch = rank // self.cp_size  # 0 = uncond, 1 = cond (the reference's batch order, guiders.py:54)
        # every rank must create every group (torch.distributed.new_group is collective over the world)
        cp_groups = [dist.new_group(ranks=list(range(b * self.cp_size, (b + 1) * self.cp_size))) for b in range(2)]
        pair_groups = [dist.new_group(ranks=[i, i + self.cp_size]) for i in range(self.cp_size)]
        self.cp = ContextParallel(cp_groups[self.branch]) if self.cp_size > 1 else None
        self.pair_group = pair_groups[rank % self.cp_size]

    def gather_branches(self, v_mine):
        """[1, ...] velocity of this rank's branch -> [2, ...] = (uncond, cond) on every rank."""
        out = torch.empty((2,) + tuple(v_mine.shape[1:]), device=v_mine.device, dtype=v_mine.dtype)
        dist.all_gather_into_tensor(out, v_mine.contiguous(), group=self.pair_group)  # group rank 0 = uncond half
        return out
