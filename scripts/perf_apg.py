"""APG guidance (scail_b200.guidance.APG): kernel cost and sampler cost.  Prints one JSON line per result with the card's
name and power limit; OUT=<dir> also appends them to <dir>/perf_apg.jsonl (nothing is written otherwise).

  kernels: ms and GB/s at the 512x512, 480x832 and 512x896 latents (21 latent frames) against 3.35 TB/s, each launch timed
           after an L2 flush, best of ROUNDS rounds of the mean over ITERS launches (perf_unipc.cold_ms):
             apg_reduce        pass 1 on the CFG pair, without momentum (reads x and the pair) and with it (also reads and
                               writes the fp32 average);
             apg_finish        pass 2, one warp per frame;
             apg_update        the Euler form in place (reads x and the pair, writes x), the momentum form (reads x, c and
                               the average, writes x), and the data-prediction form (reads x and the pair, writes D_g);
             unipc_2_dpred     the UniPC order-2 step reading D_g (reads x, x_last, D_g and 2 slots; writes x, x_last and one
                               slot);
           against cfg_euler_ (the vanilla step) and the CFG-Zero* path (its s* reduction and scaled Euler step).
  steps:   steps/s of bench.py's 14B model at 512x512 (40 blocks, CFG batch 2) over STEPS eager sampler_step calls,
           guidance=None against APG(0.5, 10.0, -0.5), the two arms alternating in each of ROUNDS rounds.
PARTS=kernels,steps selects parts (default both)."""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import perf_unipc  # noqa: E402
from perf_fp8 import card  # noqa: E402
from scail_b200 import ops, sampler, unipc  # noqa: E402
from scail_b200.guidance import APG, CFGZeroStar  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
STEPS = int(os.environ.get("STEPS", 5))
PARTS = os.environ.get("PARTS", "kernels,steps").split(",")
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
LATENTS = perf_unipc.LATENTS


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_apg.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def _row(name, shape, kernel, nbytes, ms, rounds):
    return {"part": "kernels", "latent": name, "shape": list(shape), "kernel": kernel, "ms_best": round(ms, 4),
            "ms_rounds": [round(r, 4) for r in rounds], "bytes": nbytes, "GB_per_s": round(nbytes / ms / 1e6, 1),
            "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)}


def kernels():
    sig = unipc.check_schedule(sampler.make_flow_timesteps(50, 5.0))
    i = 25
    k = unipc.step_coefficients(sig, i, 2)
    coef = [float(c) for c in torch.tensor([k.x_last_c, *k.slot_c, 0.0, k.m_c, k.y_c, *k.slot_p, 0.0, k.m_p])]
    for name, shape in LATENTS.items():
        n, T = 1, shape[1]
        for s in shape:
            n *= s
        x, xl, avg, m = (torch.randn(shape, device="cuda") for _ in range(4))
        v = torch.randn(2, *shape[1:], device="cuda").to(torch.bfloat16)
        slots = torch.randn(2, n, device="cuda")
        partials = torch.empty(ops.apg_partials_len(T), device="cuda")
        sums = torch.zeros(T, 4, device="cuda", dtype=torch.float64)
        factors = torch.zeros(T, 2, device="cuda")
        ops.apg_reduce(x, v, 0.5, partials)
        ops.apg_finish(partials, sums, factors, 10.0, T, n)
        # x, the average and the slots change over the repeated in-place launches; finite or not, the cost is the same
        for kern, nbytes, fn in (
                ("apg_reduce", n * 8, lambda: ops.apg_reduce(x, v, 0.5, partials)),
                ("apg_reduce_momentum", n * 16, lambda: ops.apg_reduce(x, v, 0.5, partials, avg, -0.5)),
                ("apg_finish", 3 * T * ops.APG_MAX_CTAS_PER_FRAME * 4,
                 lambda: ops.apg_finish(partials, sums, factors, 10.0, T, n)),
                ("apg_update_euler", n * 12, lambda: ops.apg_update_(x, v, factors, 4.0, 0.5, 0.5, 0.48)),
                ("apg_update_euler_momentum", n * 14, lambda: ops.apg_update_(x, v, factors, 4.0, 0.5, 0.5, 0.48, avg=avg)),
                ("apg_update_dpred", n * 12, lambda: ops.apg_update_(x, v, factors, 4.0, 0.5, 0.5, out=m)),
                ("unipc_2_dpred", n * (4 + 4 + 4 + 4 * 2) + n * 12,
                 lambda: ops.unipc_step_dpred_(x, xl, m, slots, k.write, coef, True)),
                ("cfg_euler", n * 12, lambda: ops.cfg_euler_(x, v, 4.0, -0.02))):
            ms, r = perf_unipc.cold_ms(fn)
            emit(_row(name, shape, kern, nbytes, ms, r))
        g = CFGZeroStar(0)
        s = g.scale(v)
        ms, r = perf_unipc.cold_ms(lambda: g.scale(v))
        emit(_row(name, shape, "cfg_zero_scale (pass 1 + pass 2)", n * 4, ms, r))
        ms, r = perf_unipc.cold_ms(lambda: ops.cfg_euler_(x, v, 4.0, -0.02, u_scale=s))
        emit(_row(name, shape, "cfg_euler_scaled", n * 12, ms, r))
        del x, xl, avg, m, v, slots, g, s
        torch.cuda.empty_cache()


def steps():
    import bench
    m = bench.build_model("cuda")
    h = bench.synthetic_inputs()
    dv = {k: v.cuda() for k, v in h.items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    uc = dict(crossattn=dv["context_uncond"])
    sig = sampler.make_flow_timesteps(50, 5.0)
    arms = {"none": None, "apg": APG(0.5, 10.0, -0.5)}

    def run(g, n):
        x = dv["x"].clone()
        if g is not None:
            g.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, guidance=g)
        torch.cuda.synchronize()
        return n / (time.perf_counter() - t0), x

    outs = {name: run(g, 2)[1] for name, g in arms.items()}  # warm-up of both update paths
    diff = float((outs["apg"] - outs["none"]).abs().max())
    res = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for name, g in arms.items():
            res[name].append(round(run(g, STEPS)[0], 5))
    med = {k: statistics.median(v) for k, v in res.items()}
    emit({"part": "steps", "workload": "SCAIL-14B, 40 blocks, latent 21x64x64 (512x512), CFG batch 2, eager sampler_step",
          "steps": STEPS, "rounds": ROUNDS, "steps_per_s": res, "median_steps_per_s": med,
          "apg_over_none_median": round(med["apg"] / med["none"] - 1, 5),
          "spread": {k: round((max(v) - min(v)) / min(v), 5) for k, v in res.items()},
          "max_abs_latent_difference_after_2_steps": diff})


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_apg.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
        if "steps" in PARTS:
            steps()
