"""CFG cache (scail_b200.cfg_cache): kernel cost, the cost of full and conditional-only steps of the 14B model, its extra
memory, and final-latent error.  Prints one JSON line per result with the card's name and power limit; OUT=<dir> also
appends them to <dir>/perf_cfg_cache.jsonl (nothing is written otherwise).

  kernels: us and GB/s of cfg_cache_delta, cfg_euler_cached_ and unipc_step_cached_ (order 2, two active slots) at the
           512x512, 480x832 and 512x896 latents (21 latent frames), beside the pair kernels cfg_euler_ and unipc_step_;
           each launch timed after an L2 flush, best of ROUNDS rounds of the mean over ITERS launches, against 3.35 TB/s.
  steps:   ms per step of bench.py's 14B model and inputs (40 blocks), eager (sampler_step) and GraphedStep, dense and
           window 2, at 512x512 and 512x896.  Arms, alternating in each of ROUNDS rounds of STEPS steps: (a) no cache,
           (b) CFGCache at threshold 0 (every step full), (c) the same cache at threshold inf (every step conditional-only).
           Reports the medians, b / a - 1 against a's run-to-run spread, c / b, whether a's and b's latents stay
           bit-identical, and the extra memory: the two fp32 delta buffers and the b = 1 workspace (of the cache's stream
           when eager, of GraphedStep's b = 1 graph when graphed).
  error:   the final latent of a 50-step sample with a fixed forced pattern (full steps 0-5 and every third step after,
           conditional-only otherwise), rel-L2 against no cache, Euler and UniPC order 2, on the small random-weight model of
           perf_forecast_cache.py.  Random weights: a report, not a quality claim.
Taylor forecast (CFGCache(order >= 1)), parts not run by default:
  fc_kernels: us and GB/s of cfg_cache_delta_forecast, cfg_euler_cached_forecast_ and unipc_step_cached_forecast_ (UniPC
           order 2) with 1, 2 and 3 active delta slots at the three latents, timed as in kernels.
  fc_steps: as steps, dense attention, with the arms (a) no cache, (b) CFGCache(0, order=2) (every step full), (c) a
           CFGCache(inf) of order 0 and (d) one of order 2, both every step conditional-only.  Reports b / a - 1 and d / c - 1
           against the spreads, and whether a's and b's latents stay bit-identical.
  fc_error: the error part at orders 0, 1 and 2.
PARTS=kernels,steps,error selects parts (default all three); RES=512x512,512x896 and MODES=dense,window2 narrow steps;
GRAPHED=0,1 narrows fc_steps to eager (0) or GraphedStep (1)."""
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
from perf_forecast_cache import small_model  # noqa: E402
from scail_b200 import cfg_cache, dit, ops, sampler, unipc  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
STEPS = int(os.environ.get("STEPS", 2))
ITERS = int(os.environ.get("ITERS", 50))
PARTS = os.environ.get("PARTS", "kernels,steps,error").split(",")
RES = os.environ.get("RES", "512x512,512x896").split(",")
MODES = os.environ.get("MODES", "dense,window2").split(",")
GRAPHED = [g == "1" for g in os.environ.get("GRAPHED", "0,1").split(",")]  # fc_steps: 0 eager, 1 GraphedStep
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
LATENTS = {"512x512": (1, 21, 16, 64, 64), "480x832": (1, 21, 16, 60, 104), "512x896": (1, 21, 16, 64, 112)}
NOTE = "random weights: a report of the error of a forced pattern against no cache, not a quality claim"


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_cfg_cache.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def cold_ms(fn):
    """Each launch timed on its own with events, after a 256 MB write that evicts the 50 MB L2 (as in a sampler step, where
    the forward in between evicts the latent).  Best of ROUNDS rounds of the mean over ITERS."""
    flush = torch.empty(64 << 20, device="cuda", dtype=torch.float32)
    res = []
    for _ in range(ROUNDS):
        fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(ITERS)]
        for s, e in ev:
            flush.zero_()
            s.record()
            fn()
            e.record()
        torch.cuda.synchronize()
        res.append(sum(s.elapsed_time(e) for s, e in ev) / ITERS)
    return min(res), res


def kernels():
    sig = unipc.check_schedule(sampler.make_flow_timesteps(50, 5.0))
    k = unipc.step_coefficients(sig, 25, 2)
    coef = [float(c) for c in torch.tensor([k.x_last_c, *k.slot_c, 0.0, k.m_c, k.y_c, *k.slot_p, 0.0, k.m_p])]
    for name, shape in LATENTS.items():
        n = math.prod(shape)
        x, xl = torch.randn(shape, device="cuda"), torch.randn(shape, device="cuda")
        v = torch.randn(2, *shape[1:], device="cuda").to(torch.bfloat16)
        c = v[1:2].contiguous()
        d_ref, d_new = torch.randn(shape, device="cuda"), torch.empty(shape, device="cuda")
        partials = torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda")
        out = torch.zeros(4, device="cuda", dtype=torch.float64)
        slots = torch.randn(2, n, device="cuda")
        # bytes moved: fp32 = 4 n, bf16 = 2 n per tensor; the UniPC steps read x, x_last and both slots, write x, x_last, a slot
        arms = {
            "cfg_cache_delta": (lambda: ops.cfg_cache_delta(v, d_ref, d_new, partials, out), n * (4 + 4 + 4)),
            "cfg_euler_cached": (lambda: ops.cfg_euler_cached_(x, c, d_ref, 4.0, -1e-3), n * (4 + 2 + 4 + 4)),
            "cfg_euler (pair)": (lambda: ops.cfg_euler_(x, v, 4.0, -1e-3), n * (4 + 4 + 4)),
            "unipc_step_cached": (lambda: ops.unipc_step_cached_(x, xl, c, d_ref, slots, k.write, 4.0, sig[25], coef, True),
                                  n * (4 + 2 + 4 + 4 + 8 + 12)),
            "unipc_step (pair)": (lambda: ops.unipc_step_(x, xl, v, slots, k.write, 4.0, sig[25], coef, True),
                                  n * (4 + 4 + 4 + 8 + 12)),
        }
        for kname, (fn, nbytes) in arms.items():
            ms, rounds = cold_ms(fn)
            emit({"part": "kernels", "kernel": kname, "latent": name, "shape": list(shape), "us_best": round(ms * 1e3, 2),
                  "us_rounds": [round(r * 1e3, 2) for r in rounds], "bytes": nbytes,
                  "GB_per_s": round(nbytes / ms / 1e6, 1), "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)})
        del x, xl, v, c, d_ref, d_new, slots
        torch.cuda.empty_cache()


def _inputs(bench, res):
    h, w = {"512x512": (64, 64), "512x896": (64, 112)}[res]
    bench.T_LAT, bench.H_LAT, bench.W_LAT = 21, h, w
    dv = {k: v.cuda() for k, v in bench.synthetic_inputs().items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    return dv["x"], cond, dict(crossattn=dv["context_uncond"])


def _runner(m, x, cond, uc, sig, graphed, c):
    if graphed:
        g = sampler.GraphedStep(m, x, cond, uc, 4.0, cfg_cache=c)
        return lambda i: g(sig[i], sig[i + 1]), g
    return lambda i: sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, cfg_cache=c), None


def _b1_workspace_bytes(c, g, dev):
    """The b = 1 workspace: the cache's stream's (eager) or the one GraphedStep's b = 1 graph holds."""
    if g is not None:
        return sum(b.numel() * b.element_size() for b in g._ws1)
    s = c.stream(dev).cuda_stream
    return sum(b.numel() * b.element_size() for k, b in dit._WS.bufs.items() if k[0][1] == s)


def steps():
    import bench
    assert STEPS >= 2, "the first round needs two full steps before the cache holds a finite indicator"
    m = bench.build_model("cuda")
    sig = sampler.make_flow_timesteps(50, 5.0)
    ad = m.mixins["adaln_layer"]
    for res in RES:
        x0, cond, uc = _inputs(bench, res)
        for mode in MODES:
            ad.attention_window = None if mode == "dense" else int(mode.replace("window", ""))
            for graphed in (False, True):
                c = cfg_cache.CFGCache(0.0)
                xa, xb = x0.clone(), x0.clone()
                run_a, ga = _runner(m, xa, cond, uc, sig, graphed, None)
                run_b, gb = _runner(m, xb, cond, uc, sig, graphed, c)
                # warm-up of every path (the first conditional-only forward allocates the b = 1 workspace), then both
                # latents restart from x0 with an empty cache
                run_a(5)
                for i, th in ((5, 0.0), (6, 0.0), (7, math.inf)):
                    c.threshold = th
                    run_b(i)
                assert [s for _, s in c.history] == [False, False, True], c.history
                torch.cuda.synchronize()
                xa.copy_(x0), xb.copy_(x0)
                c.reset()
                arms = {"a_no_cache": [], "b_threshold_0": [], "c_cond_only": []}
                equal, i = None, 10
                for r in range(ROUNDS):
                    for arm, run, th in (("a_no_cache", run_a, None), ("b_threshold_0", run_b, 0.0),
                                         ("c_cond_only", run_b, math.inf)):
                        if th is not None:
                            c.threshold = th
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        for k in range(STEPS):
                            run(i + k)
                        torch.cuda.synchronize()
                        arms[arm].append(round((time.perf_counter() - t0) * 1000.0 / STEPS, 2))
                        if r == 0 and arm == "b_threshold_0":  # a and b ran the same full steps from x0
                            equal = bool(torch.equal(xa, xb))
                    i = 10 + (i + STEPS - 10) % 30
                pattern = [s for _, s in c.history]
                assert pattern == ([False] * STEPS + [True] * STEPS) * ROUNDS, pattern
                med = {k: statistics.median(v) for k, v in arms.items()}
                spread = lambda v: round((max(v) - min(v)) / min(v), 5)
                emit({"part": "steps", "latent": res, "attention": mode, "graphed": graphed, "ms_per_step": arms,
                      "median_ms": med, "b_over_a_median": round(med["b_threshold_0"] / med["a_no_cache"] - 1, 5),
                      "a_spread": spread(arms["a_no_cache"]), "b_spread": spread(arms["b_threshold_0"]),
                      "c_over_b_median": round(med["c_cond_only"] / med["b_threshold_0"], 4),
                      "latents_a_b_bit_identical": equal,
                      "extra_bytes": {"delta_buffers": c.buffers.nbytes(), "b1_workspace": _b1_workspace_bytes(c, gb, x0.device)},
                      "rounds": ROUNDS, "steps_per_round": STEPS,
                      "workload": f"SCAIL-14B, 40 blocks, latent 21x{res}/8, CFG batch 2; {'GraphedStep' if graphed else 'eager'}"})
                del run_a, run_b, ga, gb, c
                dit._WS.bufs.clear()  # drop the b = 2 workspaces of this configuration (~11 GB each at 512x896)
                torch.cuda.empty_cache()
        ad.attention_window = None


def full(i):
    """The fixed forced pattern: full steps 0-5 and every third step after, conditional-only otherwise (29 of 50)."""
    return i <= 5 or i % 3 == 0


def error():
    m, x0, cond, uc = small_model()
    sig = sampler.make_flow_timesteps(50, 5.0)
    out = {}
    for name, order in (("euler", None), ("unipc_2", 2)):
        mk = lambda: unipc.UniPC(order) if order else None
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=50, solver=mk())
        c, s = cfg_cache.CFGCache(0.0), mk()
        if s is not None:
            s.begin(sig)
        x = x0.clone()
        for i in range(50):
            c.threshold = 0.0 if full(i) else math.inf
            sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, solver=s, cfg_cache=c)
        assert [not co for _, co in c.history] == [full(i) for i in range(50)]
        out[name] = float((x - plain).norm() / plain.norm())
    emit({"part": "error", "model": "small: 4 blocks, hidden 512, latent 5x32x32", "cond_only_steps": sum(not full(i) for i in range(50)),
          "pattern": "full steps 0-5 and every third step after", "final_latent_rel_l2_vs_no_cache": out, "note": NOTE})
    del m
    torch.cuda.empty_cache()


def fc_kernels():
    sig = unipc.check_schedule(sampler.make_flow_timesteps(50, 5.0))
    k = unipc.step_coefficients(sig, 25, 2)
    coef = [float(c) for c in torch.tensor([k.x_last_c, *k.slot_c, 0.0, k.m_c, k.y_c, *k.slot_p, 0.0, k.m_p])]
    for name, shape in LATENTS.items():
        n = math.prod(shape)
        x, xl = torch.randn(shape, device="cuda"), torch.randn(shape, device="cuda")
        v = torch.randn(2, *shape[1:], device="cuda").to(torch.bfloat16)
        c = v[1:2].contiguous()
        dslots = torch.randn(3, *shape, device="cuda")
        partials = torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda")
        out = torch.zeros(4, device="cuda", dtype=torch.float64)
        slots = torch.randn(2, n, device="cuda")
        for n_act in (1, 2, 3):
            dc = [1.0, 0.0, 0.0] if n_act == 1 else [-1.0, 2.0, 0.0] if n_act == 2 else [1.0, -3.0, 3.0]
            # bytes: fp32 = 4 n, bf16 = 2 n per tensor; each active delta slot is read once
            arms = {
                "cfg_cache_delta_forecast": (lambda: ops.cfg_cache_delta_forecast(v, dslots, 2, dc, partials, out),
                                             n * (4 + 4 * n_act + 4)),
                "cfg_euler_cached_forecast": (lambda: ops.cfg_euler_cached_forecast_(x, c, dslots, dc, 4.0, -1e-3),
                                              n * (4 + 2 + 4 * n_act + 4)),
                "unipc_step_cached_forecast": (lambda: ops.unipc_step_cached_forecast_(x, xl, c, dslots, dc, slots, k.write,
                                                                                       4.0, sig[25], coef, True),
                                               n * (4 + 2 + 4 * n_act + 4 + 8 + 12)),
            }
            for kname, (fn, nbytes) in arms.items():
                ms, rounds = cold_ms(fn)
                emit({"part": "fc_kernels", "kernel": kname, "active_slots": n_act, "latent": name, "shape": list(shape),
                      "us_best": round(ms * 1e3, 2), "us_rounds": [round(r * 1e3, 2) for r in rounds], "bytes": nbytes,
                      "GB_per_s": round(nbytes / ms / 1e6, 1),
                      "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)})
        del x, xl, v, c, dslots, slots
        torch.cuda.empty_cache()


def fc_steps():
    import bench
    assert STEPS >= 1
    m = bench.build_model("cuda")
    sig = sampler.make_flow_timesteps(50, 5.0)
    for res in RES:
        x0, cond, uc = _inputs(bench, res)
        for graphed in GRAPHED:
            c0, c2 = cfg_cache.CFGCache(0.0), cfg_cache.CFGCache(0.0, order=2)
            xa, xb = x0.clone(), x0.clone()
            run_a, ga = _runner(m, xa, cond, uc, sig, graphed, None)
            run_b, gb = _runner(m, xb, cond, uc, sig, graphed, c2)
            if graphed:  # the graphs do not depend on the cache object, so one GraphedStep serves both caches
                def run_bc(i, cache):
                    gb.cfg_cache = cache
                    gb(sig[i], sig[i + 1])
            else:
                run_bc = lambda i, cache: sampler.sampler_step(m, xb, sig[i], sig[i + 1], cond, uc, 4.0, cfg_cache=cache)
            run_a(5)
            for cache in (c0, c2):  # warm-up of every path; each cache then holds two full steps
                for i, th in ((5, 0.0), (6, 0.0), (7, math.inf)):
                    cache.threshold = th
                    run_bc(i, cache)
                assert [s for _, s in cache.history] == [False, False, True], cache.history
            torch.cuda.synchronize()
            xa.copy_(x0), xb.copy_(x0)
            c2.reset()
            arms = {"a_no_cache": [], "b_order2_threshold_0": [], "c_order0_cond_only": [], "d_order2_cond_only": []}
            equal, i = None, 10
            for r in range(ROUNDS):
                for arm, cache, th in (("a_no_cache", None, None), ("b_order2_threshold_0", c2, 0.0),
                                       ("c_order0_cond_only", c0, math.inf), ("d_order2_cond_only", c2, math.inf)):
                    if cache is not None:
                        cache.threshold = th
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for k in range(STEPS):
                        run_a(i + k) if cache is None else run_bc(i + k, cache)
                    torch.cuda.synchronize()
                    arms[arm].append(round((time.perf_counter() - t0) * 1000.0 / STEPS, 2))
                    if r == 0 and arm == "b_order2_threshold_0":  # a and b ran the same full steps from x0
                        equal = bool(torch.equal(xa, xb))
                i = 10 + (i + STEPS - 10) % 30
            assert all(s for _, s in c0.history[3:]), c0.history
            med = {k: statistics.median(v) for k, v in arms.items()}
            spread = lambda v: round((max(v) - min(v)) / min(v), 5)
            emit({"part": "fc_steps", "latent": res, "attention": "dense", "graphed": graphed, "ms_per_step": arms,
                  "median_ms": med, "spread": {k: spread(v) for k, v in arms.items()},
                  "b_over_a_median": round(med["b_order2_threshold_0"] / med["a_no_cache"] - 1, 5),
                  "d_over_c_median": round(med["d_order2_cond_only"] / med["c_order0_cond_only"] - 1, 5),
                  "latents_a_b_bit_identical": equal, "delta_slot_bytes": c2.buffers.nbytes(),
                  "rounds": ROUNDS, "steps_per_round": STEPS,
                  "workload": f"SCAIL-14B, 40 blocks, latent 21x{res}/8, CFG batch 2; {'GraphedStep' if graphed else 'eager'}"})
            del run_a, run_b, run_bc, ga, gb, c0, c2
            dit._WS.bufs.clear()
            torch.cuda.empty_cache()


def fc_error():
    m, x0, cond, uc = small_model()
    sig = sampler.make_flow_timesteps(50, 5.0)
    out = {}
    for name, sorder in (("euler", None), ("unipc_2", 2)):
        mk = lambda: unipc.UniPC(sorder) if sorder else None
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=50, solver=mk())
        for order in (0, 1, 2):
            c, s = cfg_cache.CFGCache(0.0, order=order), mk()
            if s is not None:
                s.begin(sig)
            x = x0.clone()
            for i in range(50):
                c.threshold = 0.0 if full(i) else math.inf
                sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, solver=s, cfg_cache=c)
            assert [not co for _, co in c.history] == [full(i) for i in range(50)]
            out[f"{name}_order{order}"] = float((x - plain).norm() / plain.norm())
    emit({"part": "fc_error", "model": "small: 4 blocks, hidden 512, latent 5x32x32", "cond_only_steps": sum(not full(i) for i in range(50)),
          "pattern": "full steps 0-5 and every third step after", "final_latent_rel_l2_vs_no_cache": out, "note": NOTE})
    del m
    torch.cuda.empty_cache()


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_cfg_cache.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
        if "error" in PARTS:
            error()
        if "steps" in PARTS:
            steps()
        if "fc_kernels" in PARTS:
            fc_kernels()
        if "fc_error" in PARTS:
            fc_error()
        if "fc_steps" in PARTS:
            fc_steps()
