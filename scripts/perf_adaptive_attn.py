"""Content-adaptive block-sparse self-attention (sparse.AdaptiveTiles) against dense, on one GPU.  Prints one JSON line with
the card's name and power limit; OUT=<dir> also appends it to <dir>/perf_adaptive_attn.jsonl (nothing is written otherwise).

  kernels:   at b = 2, 40 heads and N = 27 904 (512 x 512) and 48 832 (512 x 896), bf16 and fp8: ms per launch of the dense
             kernel and of the per-(batch, head) sparse kernel on maps the device selection chose with max_tiles set to land
             near densities 0.2, 0.3 and 0.5 (random Q and K give diffuse attention, so a mass threshold alone lists nearly
             every tile: the cap is what fixes the density), and ms of pooling + selection alone.  The arms alternate inside
             each round; each number is the best of REPS rounds (default 3) of 5 timed launches.
  densities: the density the selection reaches at mass 0.9, 0.95 and 0.99 (no cap) over every layer of one forward of
             bench.py's random 14B model at 512 x 512.  Random weights: this says nothing about real weights.
  steps:     sampler steps/s of bench.py's 14B model and inputs (512 x 512), the same instance toggled dense / adaptive at
             (STEP_MASS, STEP_CAP) (default 0.9, 50), alternated ROUNDS times (default 2), and the rel-L2 of the adaptive
             guided velocity against the dense one (random weights: not a statement about visual quality).
PARTS=kernels,densities,steps selects the parts."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scail_b200 import ops, sparse  # noqa: E402

TARGETS = (0.2, 0.3, 0.5)
REPS = int(os.environ.get("REPS", 3))


def timeit(fn, iters=5):
    fn(); fn(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def density(ptr):
    B, H, n1 = ptr.shape
    return float(ptr[..., -1].double().sum()) / (B * H * (n1 - 1) ** 2)


def kernels():
    B, H, d = 2, 40, 5120
    res = []
    for t, h, w in ((21, 64, 64), (21, 64, 112)):
        n_ref = (h // 2) * (w // 2)
        N = n_ref + t * n_ref + t * (h // 4) * (w // 4)
        n = -(-N // 128)
        n_forced = -(-n_ref // 128) + 1
        torch.manual_seed(0)
        qkv = torch.randn(B * N, 3 * d, device="cuda", dtype=torch.bfloat16)
        out = torch.empty(B * N, d, device="cuda", dtype=torch.bfloat16)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        Lp = ops.fp8_pad(N)
        q8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
        k8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
        w1 = torch.ones(d, device="cuda", dtype=torch.bfloat16)
        ops.rmsnorm_rope(qkv, N, d, [(0, w1), (d, w1)], out_fp8=[q8, k8])
        vt, vs = ops.quant_vt_fp8(v, B, H, N)
        ws = {}
        buf = lambda name, shape, dtype: ws.setdefault(name, torch.empty(shape, device="cuda", dtype=dtype))
        caps = {tg: max(0, round(tg * n) - n_forced) for tg in TARGETS}
        maps, dens = {}, {}
        for tg, cap in caps.items():  # maps chosen once per cap, kept for the timed launches
            for dt, (qq, kk, qs, ks) in (("bf16", (q, k, None, None)), ("fp8", (q8[0], k8[0], q8[1], k8[1]))):
                ptr, idx = sparse.AdaptiveTiles(1.0, cap).select(qq, kk, B, H, N, n_ref, buf, q_scale=qs, k_scale=ks)
                maps[(dt, tg)] = (ptr.clone(), idx.clone())
                dens[f"{dt}_{tg}"] = round(density(ptr), 4)
        sel = sparse.AdaptiveTiles(0.9)
        arms = {"bf16_dense": lambda: ops.attention(q, k, v, out, B, H, N, N),
                "fp8_dense": lambda: ops.attention_fp8(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H, N),
                "bf16_pool_select": lambda: sel.select(q, k, B, H, N, n_ref, buf),
                "fp8_pool_select": lambda: sel.select(q8[0], k8[0], B, H, N, n_ref, buf, q_scale=q8[1], k_scale=k8[1])}
        for tg in TARGETS:
            pb, ib = maps[("bf16", tg)]
            pf, i_f = maps[("fp8", tg)]
            arms[f"bf16_{tg}"] = lambda pb=pb, ib=ib: ops.attention_sparse_bh(q, k, v, out, B, H, N, pb, ib)
            arms[f"fp8_{tg}"] = lambda pf=pf, i_f=i_f: ops.attention_fp8_sparse_bh(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H,
                                                                                   N, pf, i_f)
        ms = {a: [] for a in arms}
        for _ in range(REPS):
            for a, fn in arms.items():
                ms[a].append(round(timeit(fn), 3))
        best = {a: min(x) for a, x in ms.items()}
        row = dict(N=N, latent=f"{t}x{h}x{w}", n_tiles=n, caps=caps, density=dens, ms=ms, best_ms=best)
        for dt in ("bf16", "fp8"):
            # time per listed tile pair relative to dense: 1.0 means the sparse launch runs as fast per tile as the dense one
            row[f"{dt}_time_over_density"] = {tg: round(best[f"{dt}_{tg}"] / best[f"{dt}_dense"] / dens[f"{dt}_{tg}"], 3)
                                              for tg in TARGETS}
            row[f"{dt}_pool_select_over_dense"] = round(best[f"{dt}_pool_select"] / best[f"{dt}_dense"], 4)
        res.append(row)
        del qkv, out, q8, k8, vt, vs, arms, maps, ws
        torch.cuda.empty_cache()
    return res


def bench_setup():
    import bench
    dev = torch.device("cuda", torch.cuda.current_device())
    model = bench.build_model(dev)
    host = bench.synthetic_inputs()
    d = {k: v.to(dev) for k, v in host.items()}
    cond = dict(crossattn=d["context_cond"], ref_concat=d["ref_concat"], concat_smpl_render=d["concat_smpl_render"],
                image_clip_features=d["image_clip_features"])
    return bench, model, d, cond, dict(crossattn=d["context_uncond"])


def densities(setup):
    from scail_b200 import sampler
    bench, model, d, cond, uc = setup
    ad = model.mixins["adaln_layer"]
    sig = sampler.make_flow_timesteps(50, 5.0)
    res = {}
    with torch.no_grad():
        for mass in (0.9, 0.95, 0.99):
            ad.attention_adaptive = sparse.AdaptiveTiles(mass)
            sparse.RECORD = []
            try:
                sampler.guided_velocity(model, d["x"], sig[10], cond, uc, 4.0)
                per_layer = [density(p) for p, _ in sparse.RECORD]
            finally:
                sparse.RECORD = None
                ad.attention_adaptive = None
            res[str(mass)] = dict(mean=round(sum(per_layer) / len(per_layer), 4), min=round(min(per_layer), 4),
                                  max=round(max(per_layer), 4))
    return dict(latent=f"{bench.T_LAT}x{bench.H_LAT}x{bench.W_LAT}", note="random weights: says nothing about real weights",
                density_at_mass=res)


def steps(setup):
    from scail_b200 import sampler
    bench, model, d, cond, uc = setup
    ad = model.mixins["adaln_layer"]
    adaptive = sparse.AdaptiveTiles(float(os.environ.get("STEP_MASS", 0.9)), int(os.environ.get("STEP_CAP", 50)))
    sig = sampler.make_flow_timesteps(50, 5.0)
    x = d["x"].clone()
    n_steps = int(os.environ.get("STEPS", 2))
    modes = (("dense", None), ("adaptive", adaptive))
    sps = {name: [] for name, _ in modes}
    with torch.no_grad():
        vel = {}
        for name, a in modes:
            ad.attention_adaptive = a
            vel[name] = sampler.guided_velocity(model, d["x"], sig[10], cond, uc, 4.0).clone()
            sampler.sampler_step(model, x, sig[0], sig[1], cond, uc, 4.0)  # warm-up of this mode
        for _ in range(int(os.environ.get("ROUNDS", 2))):
            for name, a in modes:
                ad.attention_adaptive = a
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(n_steps):
                    sampler.sampler_step(model, x, sig[i], sig[i + 1], cond, uc, 4.0)
                e1.record(); torch.cuda.synchronize()
                sps[name].append(round(1000.0 * n_steps / e0.elapsed_time(e1), 4))
        ad.attention_adaptive = None
    a, b = vel["dense"].double(), vel["adaptive"].double()
    return dict(latent=f"{bench.T_LAT}x{bench.H_LAT}x{bench.W_LAT}", adaptive=repr(adaptive), steps_per_round=n_steps,
                steps_per_s=sps, speedup=round(max(sps["adaptive"]) / max(sps["dense"]), 3),
                guided_velocity_rel_l2=float((b - a).norm() / a.norm()))


def main():
    assert torch.cuda.is_available(), "perf_adaptive_attn.py needs a CUDA device"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = ""
    parts = os.environ.get("PARTS", "kernels,densities,steps").split(",")
    res = dict(gpu=torch.cuda.get_device_name(), nvidia_smi=smi)
    if "kernels" in parts:
        res["kernels"] = kernels()
    if "densities" in parts or "steps" in parts:
        setup = bench_setup()
        if "densities" in parts:
            res["densities"] = densities(setup)
        if "steps" in parts:
            res["steps"] = steps(setup)
    line = json.dumps(res)
    print(line, flush=True)
    if os.environ.get("OUT"):
        os.makedirs(os.environ["OUT"], exist_ok=True)
        with open(os.path.join(os.environ["OUT"], "perf_adaptive_attn.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
