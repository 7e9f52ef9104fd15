"""Taylor forecast of the first-block residual cache (FirstBlockCache(order >= 1)) on bench.py's 14B model and inputs
(512 x 512, 40 blocks, CFG batch 2).  Prints one JSON line per result with the card's name and power limit; OUT=<dir> also
appends them to <dir>/perf_forecast_cache.jsonl (nothing is written otherwise).

  kernels: ms and GB/s of step_cache_update_slot and of step_cache_apply_forecast with 1, 2 and 3 active slots, at b = 2,
           N = 27 904 (512x512) and 48 832 (512x896), d = 5120, against 3.35 TB/s; best of ROUNDS rounds of ITERS launches.
  steps:   ms per skipped step at orders 0, 1 and 2 (all slots filled), eager (sampler_step) and GraphedStep; and a computed
           step at order 2 / threshold 0 against no cache, the two arms alternating in each of ROUNDS rounds of STEPS steps,
           with the run-to-run spread and whether the latents stay bit-identical.
  error:   the final latent of a 50-step sample with a fixed forced pattern (compute steps 0-5 and every third step after,
           skip the rest), rel-L2 against no cache, for orders 0, 1 and 2, on a small random-weight model.  error14b does
           the same on the 14B model (window 2, GraphedStep; long).  Random weights: this says nothing about visual quality
           or about the skip rate real weights allow.
PARTS=kernels,steps,error[,error14b] selects parts (default kernels,steps,error)."""
import json
import math
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from perf_fp8 import card  # noqa: E402
from scail_b200 import ops  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
STEPS = int(os.environ.get("STEPS", 2))
ITERS = int(os.environ.get("ITERS", 20))
PARTS = os.environ.get("PARTS", "kernels,steps,error").split(",")
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
WORKLOAD = "SCAIL-14B, 40 blocks, latent 21x64x64 (512x512), CFG batch 2"
NOTE = "random weights: says nothing about visual quality or about the skip rate real weights allow"


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_forecast_cache.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def best_ms(fn):
    res = []
    for _ in range(ROUNDS):
        fn(); fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(ITERS):
            fn()
        e.record()
        torch.cuda.synchronize()
        res.append(s.elapsed_time(e) / ITERS)
    return min(res), res


def kernels():
    for B, N, d, n_ref, n_seq in ((2, 27904, 5120, 1024, 21504), (2, 48832, 5120, 1792, 37632)):
        bf = torch.bfloat16
        h = torch.randn(B, N, d, device="cuda", dtype=bf)
        h1c = torch.randn(B, n_seq, d, device="cuda", dtype=bf)
        R = torch.randn(3, B, n_seq, d, device="cuda", dtype=torch.float32)
        slot = torch.ones(1, device="cuda", dtype=torch.int32)
        En = B * n_seq * d
        arms = {"update_slot": (lambda: ops.step_cache_update_slot(h, h1c, R, slot, n_ref), En * 2 * 2 + En * 4)}
        for k in (1, 2, 3):
            # small coefficients keep h finite over many in-place launches
            coef = torch.tensor([1e-3 if s < k else 0.0 for s in range(3)], device="cuda")
            arms[f"apply_forecast_{k}_slots"] = (lambda c=coef: ops.step_cache_apply_forecast(h, R, c, n_ref),
                                                 En * 2 * 2 + k * En * 4)
        for name, (fn, nbytes) in arms.items():
            ms, rounds = best_ms(fn)
            emit({"part": "kernels", "kernel": name, "B": B, "N": N, "d": d, "n_seq": n_seq, "ms_best": round(ms, 4),
                  "ms_rounds": [round(v, 4) for v in rounds], "bytes": nbytes, "GB_per_s": round(nbytes / ms / 1e6, 1),
                  "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)})
        del h, h1c, R
        torch.cuda.empty_cache()


def setup():
    import bench
    from scail_b200 import sampler
    m = bench.build_model("cuda")
    h = bench.synthetic_inputs()
    dv = {k: v.cuda() for k, v in h.items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    uc = dict(crossattn=dv["context_uncond"])
    return m, dv["x"], cond, uc, sampler.make_flow_timesteps(50, 5.0)


def _runner(m, x, cond, uc, sig, graphed, c):
    from scail_b200 import sampler
    if graphed:
        g = sampler.GraphedStep(m, x, cond, uc, 4.0, step_cache=c)
        return lambda i: g(sig[i], sig[i + 1]), g
    return lambda i: sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=c), None


def steps(m, x0, cond, uc, sig):
    from scail_b200.step_cache import FirstBlockCache
    for graphed in (False, True):
        # (1) a skipped step at orders 0, 1, 2, after order + 1 computed steps (every slot in use)
        skip_ms = {}
        for order in (0, 1, 2):
            c = FirstBlockCache(0.0, order=order)
            x = x0.clone()
            run, g = _runner(m, x, cond, uc, sig, graphed, c)
            for i in range(order + 1):
                run(10 + i)
            c.threshold = math.inf
            run(10 + order + 1)  # warm-up of the skip path
            torch.cuda.synchronize()
            res, i = [], 12 + order
            for _ in range(ROUNDS):
                t0 = time.perf_counter()
                for k in range(STEPS):
                    run(i + k)
                torch.cuda.synchronize()
                res.append(round((time.perf_counter() - t0) * 1000.0 / STEPS, 2))
                i += STEPS
            assert [s for _, s in c.history] == [False] * (order + 1) + [True] * (1 + ROUNDS * STEPS), c.history
            skip_ms[order] = res
            del c, run, g
            torch.cuda.empty_cache()
        # (2) a computed step at order 2 / threshold 0 against no cache, alternating
        c = FirstBlockCache(0.0, order=2)
        xa, xb = x0.clone(), x0.clone()
        run_a, ga = _runner(m, xa, cond, uc, sig, graphed, None)
        run_b, gb = _runner(m, xb, cond, uc, sig, graphed, c)
        run_a(10), run_b(10)
        torch.cuda.synchronize()
        res = {"a_no_cache": [], "b_order2_threshold_0": []}
        equal, i = bool(torch.equal(xa, xb)), 11
        for _ in range(ROUNDS):
            for arm, run in (("a_no_cache", run_a), ("b_order2_threshold_0", run_b)):
                t0 = time.perf_counter()
                for k in range(STEPS):
                    run(i + k)
                torch.cuda.synchronize()
                res[arm].append(round((time.perf_counter() - t0) * 1000.0 / STEPS, 2))
            equal = equal and bool(torch.equal(xa, xb))
            i += STEPS
        med = {k: statistics.median(v) for k, v in res.items()}
        emit({"part": "steps", "graphed": graphed, "skipped_ms_per_step": {f"order_{o}": v for o, v in skip_ms.items()},
              "skipped_median_ms": {f"order_{o}": statistics.median(v) for o, v in skip_ms.items()},
              "computed_ms_per_step": res, "computed_median_ms": med,
              "computed_b_over_a_median": round(med["b_order2_threshold_0"] / med["a_no_cache"] - 1, 5),
              "a_spread": round((max(res["a_no_cache"]) - min(res["a_no_cache"])) / min(res["a_no_cache"]), 5),
              "b_spread": round((max(res["b_order2_threshold_0"]) - min(res["b_order2_threshold_0"]))
                                / min(res["b_order2_threshold_0"]), 5),
              "latents_a_b_bit_identical": equal, "rounds": ROUNDS, "steps_per_round": STEPS, "workload": WORKLOAD})
        del c, run_a, run_b, ga, gb
        torch.cuda.empty_cache()


def computes(i):
    """The fixed forced pattern: compute steps 0-5 and every third step after, skip the rest (29 of 50 skipped)."""
    return i <= 5 or i % 3 == 0


def forecast_error(m, x0, cond, uc, graphed, tag):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    sig = sampler.make_flow_timesteps(50, 5.0)
    if graphed:
        x = x0.clone()
        g = sampler.GraphedStep(m, x, cond, uc, 4.0)
        for i in range(50):
            g(sig[i], sig[i + 1])
        plain = x.clone()
        del g
    else:
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=50)
    out = {}
    for order in (0, 1, 2):
        c = FirstBlockCache(0.0, order=order)
        x = x0.clone()
        run, g = _runner(m, x, cond, uc, sig, graphed, c)
        for i in range(50):
            c.threshold = 0.0 if computes(i) else math.inf
            run(i)
        assert [not s for _, s in c.history] == [computes(i) for i in range(50)]
        out[f"order_{order}"] = float((x - plain).norm() / plain.norm())
        del c, run, g
        torch.cuda.empty_cache()
    emit({"part": "error", "model": tag, "skipped_steps": sum(not computes(i) for i in range(50)),
          "pattern": "compute steps 0-5 and every third step after", "final_latent_rel_l2_vs_no_cache": out, "note": NOTE})


def small_model():
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    m = DiffusionTransformer(hidden_size=512, num_attention_heads=4, inner_hidden_size=1024, num_layers=4, text_dim=64,
                             time_embed_dim=512).to(torch.bfloat16).cuda().eval()
    g = torch.Generator().manual_seed(1)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    t, h, w = 5, 32, 32
    x0 = torch.randn(1, t, 16, h, w, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, h, w), concat_smpl_render=r(1, t, 16, h // 2, w // 2),
                image_clip_features=r(1, 257, 1280))
    return m, x0, cond, dict(crossattn=r(1, 24, 64))


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_forecast_cache.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
        if "error" in PARTS:
            forecast_error(*small_model(), graphed=False, tag="small: 4 blocks, hidden 512, latent 5x32x32")
            torch.cuda.empty_cache()
        if "steps" in PARTS or "error14b" in PARTS:
            m, x0, cond, uc, sig = setup()
            if "steps" in PARTS:
                steps(m, x0, cond, uc, sig)
            if "error14b" in PARTS:
                m.mixins["adaln_layer"].attention_window = 2
                forecast_error(m, x0, cond, uc, graphed=True, tag="14B, window 2, GraphedStep: " + WORKLOAD)
