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

from . import ops


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


def sampler_step(model, x, sigma, next_sigma, cond, uc, scale=4.0, _ctx=None, plan=None, _x_override=None, _sigma_override=None,
                 **model_kwargs):
    """One reference sampler step: x [1,t,16,h,w] fp32 (updated in place and returned).
    cond/uc: dicts with 'crossattn' [1,L,text_dim]; cond also carries ref_concat, concat_smpl_render,
    image_clip_features, concat_images (shared by both CFG branches, guiders.py:50-56).
    plan: an optional scail_b200.parallel.HybridParallel — this rank then runs ONE CFG branch (b = 1) and the two
    velocities are exchanged between partner ranks before the combine."""
    ctx = _ctx if _ctx is not None else prepare_context(cond, uc)
    kw = dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"], concat_images=cond.get("concat_images"), **model_kwargs)
    x_in = x if _x_override is None else _x_override          # guided_velocity(): forward on x_in, accumulate into a zero latent
    c_noise = float(sigma if _sigma_override is None else _sigma_override) * 1000.0  # RFScaling: c_noise = 1000 sigma
    if plan is None:
        x2 = torch.cat([x_in, x_in], 0)
        ts = torch.full((2,), c_noise, device=x.device, dtype=torch.float32)
        v = model(x2, timesteps=ts, context=ctx, **kw)
    else:
        b = plan.branch
        ts = torch.full((1,), c_noise, device=x.device, dtype=torch.float32)
        v = plan.gather_branches(model(x_in, timesteps=ts, context=ctx[b:b + 1], **kw))
    return ops.cfg_euler_(x, v.contiguous(), scale, float(next_sigma) - float(sigma))


def sample(model, x, cond, uc, num_steps=50, shift_scale=5.0, scale=4.0, plan=None):
    """RFSampler.__call__ (sampling.py:965-982): the full Euler loop.  With `adaln_layer.cache_cross_kv` the step-invariant
    conditioning (text / CLIP embeddings and all layers' cross-attention K,V) is computed once for this call."""
    sig = make_flow_timesteps(num_steps, shift_scale)
    ctx = prepare_context(cond, uc)
    cache = getattr(model.mixins["adaln_layer"], "cache_cross_kv", False) if hasattr(model, "mixins") else False
    cache = cache and plan is None  # (a CFG-parallel rank feeds its own row of ctx: a different tensor object)
    if cache:
        model.set_conditioning(ctx, cond["image_clip_features"], batch=2)
    try:
        for i in range(num_steps):
            x = sampler_step(model, x, sig[i], sig[i + 1], cond, uc, scale, _ctx=ctx, plan=plan)
    finally:
        if cache:
            model.clear_conditioning()
    return x


def guided_velocity(model, x, sigma, cond, uc, scale=4.0, ctx=None, plan=None):
    """RFSampler.denoise (sampling.py:945-953): CFG batch-2 forward + `u + s (c - u)` -> fp32 guided velocity [1,t,16,h,w]
    (the fused CFG+Euler kernel applied to a zero latent with d_sigma = 1)."""
    return sampler_step(model, torch.zeros_like(x), 0.0, 1.0, cond, uc, scale, _ctx=ctx, plan=plan, _x_override=x, _sigma_override=sigma)


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


def sample_long(model, x, cond, uc, tile_indices, num_steps=50, shift_scale=5.0, scale=4.0, denoise=None, plan=None):
    """RFSamplerLong.__call__ (sampling.py:1070-1085): tiled long-video sampling.  x [1,T,16,h,w] fp32 over ALL latent frames;
    cond['smpl_tiled'] [1, n_tiles, segment, 16, h/2, w/2] holds the pose render of every window; `tile_indices` lists the
    latent-frame indices of every window (equal lengths).  `denoise` overrides the network call (tests)."""
    sig = make_flow_timesteps(num_steps, shift_scale).to(x.device)
    smpl_tiled = cond["smpl_tiled"]
    uc = dict(uc if uc is not None else cond)
    cond = dict(cond)
    if denoise is None:
        ctx = prepare_context(cond, uc)

        def denoise(x_tile, sigma, c_k, u_k):
            return guided_velocity(model, x_tile.contiguous(), float(sigma), c_k, u_k, scale, ctx=ctx, plan=plan)
    for i in range(num_steps):
        x = sampler_step_long(denoise, x, sig[i], sig[i + 1], tile_indices, smpl_tiled, cond, uc)
    return x


class GraphedStep:
    """One sampler step with the whole CFG batch-2 DiT forward (~780 kernel launches of libscail_b200.so, SURVEY.md §8f rank 3)
    captured ONCE in a CUDA graph and replayed per step: 3 host launches per step (timestep fill, graph replay, CFG+Euler)
    instead of ~780, and none of the reference's per-layer host syncs (sat/transformer_defaults.py:56-57) by construction.
    The latent `x`, the timestep vector and the conditioning tensors are static buffers owned by this object; results are
    bit-identical to `sampler_step` (same kernels, same order).  Single-GPU path (NCCL collectives are not captured).
    The graph runs in the `fp8_linear` mode of construction time.  With fp8 it reads the e4m3 weight copies in place: every
    call first re-derives, into the same buffers, the copies of weights that changed since (e.g. after load_state_dict)."""

    def __init__(self, model, x, cond, uc, scale=4.0):
        if getattr(model.mixins["adaln_layer"], "cp", None) is not None:
            raise NotImplementedError("GraphedStep captures the single-GPU forward; use sampler_step under context parallelism")
        self.model, self.scale = model, scale
        self.x = x  # fp32 [1,t,16,h,w], updated in place every step
        dev = x.device
        self.ts = torch.zeros(2, device=dev, dtype=torch.float32)
        self.ctx = prepare_context(cond, uc)
        self.kw = dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
                       image_clip_features=cond["image_clip_features"], concat_images=cond.get("concat_images"))
        assert ops.ATTN_EVENTS is None, "event timing of individual launches cannot be captured"
        self.adaln = model.mixins["adaln_layer"]
        self.fp8 = getattr(self.adaln, "fp8_linear", False)
        # the e4m3 weights are derived on this stream and held here: the graph replays against these very buffers
        self._fp8_weights = self.adaln.prepare_fp8_weights() if self.fp8 else []
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

    def _forward(self):
        return self.model(torch.cat([self.x, self.x], 0), timesteps=self.ts, context=self.ctx, **self.kw).contiguous()

    def __call__(self, sigma, next_sigma):
        if self.fp8:
            self.adaln.prepare_fp8_weights()
        self.ts.fill_(float(sigma) * 1000.0)
        self.graph.replay()
        return ops.cfg_euler_(self.x, self.v, self.scale, float(next_sigma) - float(sigma))


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
