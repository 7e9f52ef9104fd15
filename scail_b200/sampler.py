"""Rectified-flow Euler sampler step with classifier-free guidance: the public per-step API.

Mirrors the reference call chain (paths relative to /root/reference):
  RFSampler.sampler_step / denoise      sgm/modules/diffusionmodules/sampling.py:950-963
  VanillaCFG.prepare_inputs / __call__  sgm/modules/diffusionmodules/guiders.py:41-57
  Denoiser.forward + RFScaling          denoiser.py:25-43, denoiser_scaling.py:71-79  (c_in=c_out=1, c_skip=0, c_noise=1000*sigma)
  make_flow_timesteps                   sampling.py:888-903
The latent stays fp32 across steps (diffusion_video.py:470); the DiT consumes/produces bf16.
"""
import numpy as np
import torch

from . import cfg_cache as cfgc
from . import dit, ops
from . import guidance as gd
from .step_cache import check_supported


def make_flow_timesteps(num_steps=50, shift_scale=5.0, t_start=0.0):
    s = np.linspace(t_start, 1.0, num_steps + 1, endpoint=True)
    s = s / (shift_scale + s - shift_scale * s)
    return 1 - torch.tensor(s, dtype=torch.float32)


def prepare_context(cond, uc):
    """VanillaCFG.prepare_inputs (guiders.py:47-57) for the 'crossattn' key: the batch is [uncond, cond]; when the two text
    contexts differ in length the UNCOND one is extended by repeating its last token row |Lc - Lu| times (guiders.py:52-53)
    before the concat (so, as in the reference, an uncond context longer than the cond one is an error)."""
    u, c = uc["crossattn"], cond["crossattn"]
    if u.shape[1] != c.shape[1]:
        u = torch.cat([u, u[:, -1:].repeat(1, abs(c.shape[1] - u.shape[1]), 1)], dim=1)
    return torch.cat((u, c), 0)


def _adaln(model):
    return model.mixins["adaln_layer"] if hasattr(model, "mixins") else None


def _check_cfg_cache(model, cfg_cache, plan=None, model_kwargs=None):
    """Validate a cfg_cache argument and refuse what it does not cover (scail_b200.cfg_cache.check_supported)."""
    if cfgc.check_cache(cfg_cache) is not None:
        mk = model_kwargs or {}
        cfgc.check_supported(getattr(_adaln(model), "cp", None), mk.get("chunk_dim"), mk.get("_num_layers"), plan)


def _check_guidance(model, guidance, model_kwargs=None):
    """Validate a guidance argument and refuse what it does not cover (scail_b200.guidance.check_supported)."""
    if gd.check_guidance(guidance) is not None:
        gd.check_supported(getattr(_adaln(model), "cp", None), (model_kwargs or {}).get("chunk_dim"))


def sampler_step(model, x, sigma, next_sigma, cond, uc, scale=4.0, _ctx=None, plan=None, _x_override=None, _sigma_override=None,
                 step_cache=None, solver=None, cfg_cache=None, guidance=None, **model_kwargs):
    """One reference sampler step: x [1,t,16,h,w] fp32 (updated in place and returned).
    cond/uc: dicts with 'crossattn' [1,L,text_dim]; cond also carries ref_concat, concat_smpl_render,
    image_clip_features, concat_images (shared by both CFG branches, guiders.py:50-56).
    plan: an optional scail_b200.parallel.HybridParallel — this rank then runs ONE CFG branch (b = 1) and the two
    velocities are exchanged between partner ranks before the combine.
    step_cache: an optional scail_b200.step_cache.FirstBlockCache, passed to the forward with this step's sigma (single GPU
    only).
    solver: an optional scail_b200.unipc.UniPC with a bound schedule; its step replaces the Euler update.  (sigma, next_sigma)
    must be the solver's next pair and x its latent, else ValueError before anything runs.
    cfg_cache: an optional scail_b200.cfg_cache.CFGCache (single GPU only).  It decides before the forward whether this step
    runs the conditional branch alone (b = 1, on the cache's stream) and rebuilds u = c - delta for the update (delta
    forecast at this step's sigma when the cache's order is >= 1); the first-block cache then sits the step out.
    guidance: an optional scail_b200.guidance.CFGZeroStar or APG (not under context parallelism or chunk_dim).  It counts
    this step first: a zero-initialised step runs no forward and tells neither cache about it, leaves x as it is with Euler
    and runs the solver on a zero CFG pair; any other step scales u by s*, reduced on the device from the pair (or from the
    CFG cache's rebuilt u), before the combine.  (guided_velocity does not count steps: it applies s* only.)  An APG step
    reduces its per-frame factors on the device from the same u and c and replaces the combine by its data-prediction rule:
    the Euler step, or the solver's step on D_g."""
    _check_cfg_cache(model, cfg_cache, plan, model_kwargs)
    _check_guidance(model, guidance, model_kwargs)
    if solver is not None:
        solver.check_step(x, sigma, next_sigma)
    if step_cache is not None:
        check_supported(plan=plan)
    if guidance is not None and _x_override is None and guidance.begin_step():
        return guidance.zero_step(x, scale, sigma, next_sigma, solver)
    cond_only = cfg_cache is not None and cfg_cache.begin_step(x, sigma if _sigma_override is None else _sigma_override)
    if step_cache is not None and not cond_only:
        step_cache.set_sigma(sigma if _sigma_override is None else _sigma_override)
        model_kwargs["_step_cache"] = step_cache
    ctx = _ctx if _ctx is not None else prepare_context(cond, uc)
    kw = dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"], concat_images=cond.get("concat_images"), **model_kwargs)
    x_in = x if _x_override is None else _x_override          # guided_velocity(): forward on x_in, accumulate into a zero latent
    c_noise = float(sigma if _sigma_override is None else _sigma_override) * 1000.0  # RFScaling: c_noise = 1000 sigma
    if cond_only:
        ts = torch.full((1,), c_noise, device=x.device, dtype=torch.float32)
        c = cfg_cache.cond_forward(model, x_in, ts, ctx[1:2], kw)
        return cfg_cache.cond_update(x, c, scale, sigma, next_sigma, solver, guidance)
    if plan is None:
        x2 = torch.cat([x_in, x_in], 0)
        ts = torch.full((2,), c_noise, device=x.device, dtype=torch.float32)
        v = model(x2, timesteps=ts, context=ctx, **kw)
    else:
        b = plan.branch
        ts = torch.full((1,), c_noise, device=x.device, dtype=torch.float32)
        v = plan.gather_branches(model(x_in, timesteps=ts, context=ctx[b:b + 1], **kw))
    if cfg_cache is not None:
        cfg_cache.full_step(v.contiguous())
    if guidance is not None:
        return guidance.update(x, v.contiguous(), scale, sigma, next_sigma, solver)
    if solver is not None:
        return solver.step(x, v.contiguous(), scale, sigma, next_sigma)
    return ops.cfg_euler_(x, v.contiguous(), scale, float(next_sigma) - float(sigma))


def sample(model, x, cond, uc, num_steps=50, shift_scale=5.0, scale=4.0, plan=None, step_cache=None, solver=None, cfg_cache=None,
           guidance=None):
    """RFSampler.__call__ (sampling.py:965-982): the full Euler loop.  With `adaln_layer.cache_cross_kv` the step-invariant
    conditioning (text / CLIP embeddings and all layers' cross-attention K,V) is computed once for this call.  step_cache (a
    scail_b200.step_cache.FirstBlockCache) is reset here and then decides on every step whether blocks 1..L-1 run.
    solver (a scail_b200.unipc.UniPC) is bound to this call's schedule here and replaces the Euler update on every step.
    cfg_cache (a scail_b200.cfg_cache.CFGCache) is reset here and then decides on every step whether only the conditional
    branch runs; with cache_cross_kv that forward reads the cond row of this call's conditioning.  guidance (a
    scail_b200.guidance.CFGZeroStar or APG) is reset here; a CFGZeroStar's first zero_init_steps steps run no forward, and
    an APG's momentum starts from zero."""
    _check_cfg_cache(model, cfg_cache, plan)
    _check_guidance(model, guidance)
    if guidance is not None:
        guidance.reset()
    if cfg_cache is not None:
        cfg_cache.reset()
    if step_cache is not None:
        check_supported(plan=plan)
        step_cache.reset()
    sig = make_flow_timesteps(num_steps, shift_scale)
    if solver is not None:
        solver.begin(sig)
    ctx = prepare_context(cond, uc)
    cache = getattr(model.mixins["adaln_layer"], "cache_cross_kv", False) if hasattr(model, "mixins") else False
    cache = cache and plan is None  # (a CFG-parallel rank feeds its own row of ctx: a different tensor object)
    if cache:
        model.set_conditioning(ctx, cond["image_clip_features"], batch=2)
    try:
        for i in range(num_steps):
            x = sampler_step(model, x, sig[i], sig[i + 1], cond, uc, scale, _ctx=ctx, plan=plan, step_cache=step_cache,
                             solver=solver, cfg_cache=cfg_cache, guidance=guidance)
    finally:
        if cache:
            model.clear_conditioning()
    return x


def guided_velocity(model, x, sigma, cond, uc, scale=4.0, ctx=None, plan=None, guidance=None):
    """RFSampler.denoise (sampling.py:945-953): CFG batch-2 forward + `u + s (c - u)` -> fp32 guided velocity [1,t,16,h,w]
    (the fused CFG+Euler kernel applied to a zero latent with d_sigma = 1).  With guidance (a CFGZeroStar), u is scaled by
    this call's own s* (the scaled kernel); zero-init is the caller's decision (sample_long), so no step is counted.  An
    APG is refused (NotImplementedError): its rule needs the step's latent and sigma, and this call runs on a zero latent."""
    _check_guidance(model, guidance)
    if isinstance(guidance, gd.APG):
        raise NotImplementedError("guided_velocity does not take an APG guidance: its data predictions need the step's "
                                  "latent, and guided_velocity accumulates into a zero latent; use sampler_step")
    return sampler_step(model, torch.zeros_like(x), 0.0, 1.0, cond, uc, scale, _ctx=ctx, plan=plan, _x_override=x, _sigma_override=sigma,
                        guidance=guidance)


def make_tile_indices(num_frames, segment, stride):
    """Overlapping latent-frame windows for sample_long: [0..segment), [stride..stride+segment), ... (the reference's engine takes
    `tile_indices` from its caller, diffusion_video.py:467,564-567; this helper builds the usual sliding windows)."""
    if (num_frames - segment) % stride:
        raise ValueError("num_frames - segment must be a multiple of stride so that the windows cover every frame")
    return [list(range(a, a + segment)) for a in range(0, num_frames - segment + 1, stride)]


def sampler_step_long(denoise, x, sigma, next_sigma, tile_indices, smpl_tiled, cond, uc):
    """RFSamplerLong.sampler_step (sampling.py:1027-1068): every pair of neighbouring windows (k, k+1) is denoised with its own
    pose-render tile and blended with a triangular weight over the window; the reference denoises each interior window
    twice (as `next` of pair k-1 and `current` of pair k) with identical inputs — here each window is denoised ONCE and the
    result is accumulated in exactly the reference's order, so the sums are bit-identical at half the forwards.
    denoise(x_tile, sigma, cond_tile, uc_tile) -> fp32 guided velocity."""
    denoised = torch.zeros_like(x)
    weight_sum = torch.zeros((x.shape[1],), device=x.device)
    segment_length = len(tile_indices[0])
    weight = (torch.arange(segment_length, device=x.device) + 0.5) * 2.0 / segment_length
    weight = torch.minimum(weight, 2.0 - weight)
    cache = {}

    def tile_out(k):
        if k not in cache:
            c_k, u_k = dict(cond), dict(uc)
            c_k["concat_smpl_render"] = u_k["concat_smpl_render"] = smpl_tiled[:, k]
            cache[k] = denoise(x[:, tile_indices[k]], sigma, c_k, u_k).to(torch.float32)
        return cache[k]

    for k in range(len(tile_indices) - 1):
        cur, nxt = tile_indices[k], tile_indices[k + 1]
        d_cur, d_nxt = tile_out(k), tile_out(k + 1)
        denoised[:, cur] += d_cur * weight[:, None, None, None]
        weight_sum[cur] += weight
        denoised[:, nxt] += d_nxt * weight[:, None, None, None]
        weight_sum[nxt] += weight
        cache.pop(k, None)
    denoised.div_(weight_sum[:, None, None, None])
    return x + (next_sigma - sigma) * denoised


def sample_long(model, x, cond, uc, tile_indices, num_steps=50, shift_scale=5.0, scale=4.0, denoise=None, plan=None,
                guidance=None):
    """RFSamplerLong.__call__ (sampling.py:1070-1085): tiled long-video sampling.  x [1,T,16,h,w] fp32 over ALL latent frames;
    cond['smpl_tiled'] [1, n_tiles, segment, 16, h/2, w/2] holds the pose render of every window; `tile_indices` lists the
    latent-frame indices of every window (equal lengths).  `denoise` overrides the network call (tests).
    guidance (a scail_b200.guidance.CFGZeroStar) is reset here.  On a zero-initialised step every window's velocity is zero,
    so the whole step is skipped and x is unchanged; on every other step each window's guided_velocity uses its own s*.
    An APG is refused (NotImplementedError): its momentum would need state per window."""
    _check_guidance(model, guidance)
    if isinstance(guidance, gd.APG):
        raise NotImplementedError("sample_long does not take an APG guidance: its momentum average would need state per "
                                  "window, and each window would need its own per-frame sums; use CFGZeroStar or None")
    if guidance is not None:
        guidance.reset()
    sig = make_flow_timesteps(num_steps, shift_scale).to(x.device)
    smpl_tiled = cond["smpl_tiled"]
    uc = dict(uc if uc is not None else cond)
    cond = dict(cond)
    if denoise is None:
        ctx = prepare_context(cond, uc)

        def denoise(x_tile, sigma, c_k, u_k):
            return guided_velocity(model, x_tile.contiguous(), float(sigma), c_k, u_k, scale, ctx=ctx, plan=plan,
                                   guidance=guidance)
    for i in range(num_steps):
        if guidance is not None and guidance.begin_step():
            continue
        x = sampler_step_long(denoise, x, sig[i], sig[i + 1], tile_indices, smpl_tiled, cond, uc)
    return x


class GraphedStep:
    """One sampler step with the whole CFG batch-2 DiT forward (~780 kernel launches of libscail_b200.so, SURVEY.md §8f rank 3)
    captured ONCE in a CUDA graph and replayed per step: 3 host launches per step (timestep fill, graph replay, CFG+Euler)
    instead of ~780, and none of the reference's per-layer host syncs (sat/transformer_defaults.py:56-57) by construction.
    The latent `x`, the timestep vector and the conditioning tensors are static buffers owned by this object; results are
    bit-identical to `sampler_step` (same kernels, same order).  Single-GPU path (NCCL collectives are not captured).
    The graph runs in the `fp8_linear`, `fp8_attention`, `attention_window` and `attention_adaptive` modes of construction
    time; a window's tile map is held by scail_b200.sparse for the life of the process, so the graph reads it at a fixed
    address.  attention_adaptive selects its maps on the device on every replay (tile pooling and selection are captured
    kernels writing the per-stream workspace), so they follow the replayed step's Q and K.  With fp8 it reads the e4m3 weight copies in place
    (the int8 ones with fp8_linear="int8"): every call first re-derives, into the same buffers, the copies of weights that
    changed since (e.g. after load_state_dict).
    step_cache (a scail_b200.step_cache.FirstBlockCache): the step runs as three graphs with the host's skip decision between
    them (bit-identical to sampler_step with the same cache and thresholds).  The cache is reset at construction; when its
    buffers are dropped or replaced later (reset(), another geometry) the graphs are captured again, and the next step
    computes.  At order >= 1, graphs (2) and (3) hold the forecast kernels, which read the slot and coefficients from the
    cache's control block: the host writes it between graph (1) and the tail, so the same graphs serve every step.
    solver (a scail_b200.unipc.UniPC, with a schedule bound by solver.begin): its step runs eagerly after the replay, in
    place of CFG+Euler, with its coefficients passed by value, so no graph depends on it; the step is validated before
    anything runs.
    cfg_cache (a scail_b200.cfg_cache.CFGCache, reset at construction): the conditional-only forward (b = 1 on the cond
    row) is one more graph, captured on a stream of this object's own so that it has its own workspace; the host decides
    before each step which graphs replay.  Every graph's workspace tensors are held here (_workspace_of).  The delta kernel and the updates run eagerly after the replay (delta_ref and delta_new
    alternate between two buffers, which a graph would fix; at order >= 1 the forecast coefficients are kernel arguments
    computed from each step's sigma, so no graph depends on them either).
    guidance (a scail_b200.guidance.CFGZeroStar or APG, reset at construction): a zero-initialised step replays nothing and
    runs only the solver's step on a zero pair, if there is a solver; on any other step the reduction of s* and the scaled
    update run eagerly after the replay, and s* stays on the device, so no graph depends on it.  An APG's reductions and
    update run eagerly after the replay in the same way, with sigma and its coefficients as kernel arguments."""

    def __init__(self, model, x, cond, uc, scale=4.0, step_cache=None, solver=None, cfg_cache=None, guidance=None):
        _check_cfg_cache(model, cfg_cache)
        _check_guidance(model, guidance)
        if step_cache is not None:
            check_supported(getattr(model.mixins["adaln_layer"], "cp", None))
        if getattr(model.mixins["adaln_layer"], "cp", None) is not None:
            raise NotImplementedError("GraphedStep captures the single-GPU forward; use sampler_step under context parallelism")
        self.model, self.scale, self.solver = model, scale, solver
        self.x = x  # fp32 [1,t,16,h,w], updated in place every step
        dev = x.device
        self.ts = torch.zeros(2, device=dev, dtype=torch.float32)
        self.ctx = prepare_context(cond, uc)
        self.kw = dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
                       image_clip_features=cond["image_clip_features"], concat_images=cond.get("concat_images"))
        assert ops.ATTN_EVENTS is None, "event timing of individual launches cannot be captured"
        self.adaln = model.mixins["adaln_layer"]
        self.fp8 = getattr(self.adaln, "fp8_linear", False)
        # the 8-bit weights (e4m3, or int8 for fp8_linear="int8") are derived on this stream and held here: the graph replays
        # against these very buffers
        self._w8_dtype = ops.INT8 if dit.linear_format(self.fp8) == ops.INT8 else ops.FP8
        self._fp8_weights = self.adaln.prepare_fp8_weights(dtype=self._w8_dtype) if self.fp8 else []
        self.step_cache, self.cfg_cache, self.guidance = step_cache, cfg_cache, guidance
        if guidance is not None:
            guidance.reset()
        if cfg_cache is not None:
            cfg_cache.reset()
            self._capture_cond()
        if step_cache is not None:
            step_cache.reset()
            self._capture_cached()
            return
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():  # warm-up on the capture stream: workspaces and TMA descriptors exist
            self._forward()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES
        with torch.cuda.graph(self.graph, stream=side), torch.no_grad():
            self.v = self._forward()
        self.kernels_in_graph = ops.LAUNCHES - n0
        self._ws = _workspace_of(side)

    def _forward(self):
        return self.model(torch.cat([self.x, self.x], 0), timesteps=self.ts, context=self.ctx, **self.kw).contiguous()

    def _capture_cond(self):
        """The conditional-only forward as one graph on a capture stream of its own (so its b = 1 workspace is not the b = 2
        graph's): x itself (b = 1), timesteps [1] and the cond row of the context."""
        dev = self.x.device
        self.ts1 = torch.zeros(1, device=dev, dtype=torch.float32)
        self.ctx1 = self.ctx[1:2]
        side, main = torch.cuda.Stream(device=dev), torch.cuda.current_stream(dev)
        fwd = lambda: self.model(self.x, timesteps=self.ts1, context=self.ctx1, **self.kw).contiguous()
        side.wait_stream(main)
        with torch.cuda.stream(side), torch.no_grad():  # warm-up: the capture stream's workspace and TMA descriptors exist
            fwd()
        main.wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph1 = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES
        with torch.cuda.graph(self.graph1, stream=side), torch.no_grad():
            self.v1 = fwd()
        self.kernels_in_graph1 = ops.LAUNCHES - n0
        self._ws1 = _workspace_of(side)

    def _head(self):
        return self.model.step_cache_head(self.step_cache, torch.cat([self.x, self.x], 0), timesteps=self.ts, context=self.ctx,
                                          **self.kw)

    def _capture_cached(self):
        """The first-block cache's three graphs, sharing one memory pool and replayed in capture order: (1) embeddings, patch
        embedding and block 0; (2) blocks 1..L-1, the R update and the final layer; (3) the R apply and the final layer.  The
        indicator runs between (1) and (2) or (3) outside the graphs, because its r_ref / r_new alternate between two buffers
        and a graph would fix them."""
        self.graphs = self.head = self.v_run = self.v_skip = None
        dev = self.x.device
        if getattr(self, "_side", None) is None:  # one capture stream for every (re)capture: one set of stream workspaces
            self._side = torch.cuda.Stream(device=dev)
        side = self._side
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():  # warm-up of every path: workspaces and TMA descriptors exist
            head = self._head()
            head.buffers.indicator(head.h0)
            self.model.step_cache_tail(head, False)
            self.model.step_cache_tail(head, True)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.step_cache.has_state = False  # the warm-up overwrote R: the next step computes
        graphs = [torch.cuda.CUDAGraph() for _ in range(3)]
        n0 = ops.LAUNCHES
        with torch.cuda.graph(graphs[0], stream=side), torch.no_grad():
            self.head = self._head()
        pool = graphs[0].pool()
        with torch.cuda.graph(graphs[1], stream=side, pool=pool), torch.no_grad():
            self.v_run = self.model.step_cache_tail(self.head, False).contiguous()
        with torch.cuda.graph(graphs[2], stream=side, pool=pool), torch.no_grad():
            self.v_skip = self.model.step_cache_tail(self.head, True).contiguous()
        self.graphs = graphs
        self.kernels_in_graph = ops.LAUNCHES - n0
        self._ws = _workspace_of(side)

    def _update(self, v, sigma, next_sigma):
        if self.guidance is not None:
            return self.guidance.update(self.x, v, self.scale, sigma, next_sigma, self.solver)
        if self.solver is not None:
            return self.solver.step(self.x, v, self.scale, sigma, next_sigma)
        return ops.cfg_euler_(self.x, v, self.scale, float(next_sigma) - float(sigma))

    def __call__(self, sigma, next_sigma):
        if self.solver is not None:
            self.solver.check_step(self.x, sigma, next_sigma)
        g = self.guidance
        if g is not None and g.begin_step():
            return g.zero_step(self.x, self.scale, sigma, next_sigma, self.solver)
        if self.fp8:
            self.adaln.prepare_fp8_weights(dtype=self._w8_dtype)
        cc = self.cfg_cache
        if cc is not None and cc.begin_step(self.x, sigma):
            self.ts1.fill_(float(sigma) * 1000.0)
            self.graph1.replay()
            return cc.cond_update(self.x, self.v1, self.scale, sigma, next_sigma, self.solver, g)
        v = self._full(sigma)
        if cc is not None:
            cc.full_step(v)
        return self._update(v, sigma, next_sigma)

    def _full(self, sigma):
        """Replay the b = 2 forward (with the first-block cache's decision between its graphs) -> the CFG pair."""
        self.ts.fill_(float(sigma) * 1000.0)
        if self.step_cache is None:
            self.graph.replay()
            return self.v
        sc = self.step_cache
        sc.set_sigma(sigma)
        sc.begin()
        if sc.buffers is not self.head.buffers:  # reset() or another geometry since the capture dropped the captured buffers
            self._capture_cached()
        self.graphs[0].replay()
        bufs = self.head.buffers
        bufs.indicator(self.head.h0)
        skip = sc.decide(bufs.read_indicator())
        sc.stage(skip)
        self.graphs[2 if skip else 1].replay()
        if not skip:
            sc.computed()
        return self.v_skip if skip else self.v_run


def _workspace_of(stream):
    """The DiT workspace tensors of `stream`, which a graph just captured on it reads and writes.  GraphedStep holds them:
    stream handles come from a pool and recur, so another forward on a stream with the same handle may later replace the
    workspace entries (dit._Workspace frees a buffer whose shape changes), and the graph must keep its memory."""
    h = stream.cuda_stream
    return [b for k, b in dit._WS.bufs.items() if k[0][1] == h]


class HostStep:
    """End-to-end step through host buffers: pinned host -> device copies of the step's inputs, one sampler
    step, device -> pinned host copy of the updated latent.  This is what bench.py's `e2e` times."""

    def __init__(self, model, host_inputs, device="cuda", step_fn=None, plan=None):
        self.model, self.device, self.plan = model, device, plan
        self.step_fn = step_fn or sampler_step  # bench.py's library arm passes baseline.torchlib.sampler_step
        self.host = {k: v.pin_memory() for k, v in host_inputs.items()}
        self.out_host = torch.empty_like(self.host["x"]).pin_memory()
        self.h2d_bytes = sum(v.numel() * v.element_size() for v in self.host.values())
        self.d2h_bytes = self.out_host.numel() * self.out_host.element_size()

    def __call__(self, sigma, next_sigma, scale=4.0):
        d = {k: v.to(self.device, non_blocking=True) for k, v in self.host.items()}
        cond = dict(crossattn=d["context_cond"], ref_concat=d["ref_concat"], concat_smpl_render=d["concat_smpl_render"],
                    image_clip_features=d["image_clip_features"], concat_images=None)
        kw = dict(plan=self.plan) if self.plan is not None else {}
        x = self.step_fn(self.model, d["x"], sigma, next_sigma, cond, dict(crossattn=d["context_uncond"]), scale, **kw)
        self.out_host.copy_(x, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self.out_host
