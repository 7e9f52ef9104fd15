"""Wan2.1 VAE timing and peak memory, random weights.  Defaults: decode at config 5 (latent [1,16,21,64,64] ->
[1,3,81,512,512]).  Environment: T, H, W = latent frames / height / width; CHUNK = latent frames per chunk (unset or
"none" = whole sequence); MODE = decode | encode (encode runs the matching 1+4(T-1) x 8H x 8W video); REPS = timed runs;
OUT = optional JSON-lines file the result is appended to (it is always printed)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scail_b200 import ops  # noqa: E402
from scail_b200.wan_vae import WanVAE  # noqa: E402

VAE_TFLOP_A = 180.5  # SURVEY §8d


def main():
    T, h, w = int(os.environ.get("T", 21)), int(os.environ.get("H", 64)), int(os.environ.get("W", 64))
    chunk = os.environ.get("CHUNK", "none")
    chunk = None if chunk.lower() in ("", "none") else int(chunk)
    mode = os.environ.get("MODE", "decode")
    reps = int(os.environ.get("REPS", 3))
    assert mode in ("decode", "encode"), mode
    torch.manual_seed(7)
    vae = WanVAE(dim=96)
    if mode == "decode":
        inp = torch.randn(16, T, h, w, device="cuda").to(torch.bfloat16)
        run = lambda: vae.decode([inp], chunk_frames=chunk)  # noqa: E731
    else:
        inp = torch.rand(3, 1 + 4 * (T - 1), 8 * h, 8 * w, device="cuda") * 2 - 1
        run = lambda: vae.encode([inp], chunk_frames=chunk)  # noqa: E731
    res = {"mode": mode, "latent": [T, h, w], "chunk_frames": chunk}
    with torch.no_grad():
        try:
            out = run()  # warm-up: packed weights, TMA descriptors
            torch.cuda.synchronize()
            del out
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            times = []
            for _ in range(reps):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                l0 = ops.LAUNCHES
                s.record()
                out = run()
                e.record()
                torch.cuda.synchronize()
                times.append(s.elapsed_time(e))
                launches = ops.LAUNCHES - l0
                res["out"], res["finite"] = list(out.shape), bool(torch.isfinite(out).all())
                del out
        except torch.cuda.OutOfMemoryError as err:
            res["oom"] = str(err).splitlines()[0]
            print(json.dumps(res))
            return
    ms = min(times)
    res.update({"ms": ms, "all_ms": times, "launches": launches,
                "peak_gb": torch.cuda.max_memory_allocated() / 2**30,
                "peak_act_gb": (torch.cuda.max_memory_allocated() - base) / 2**30,
                "tflops": VAE_TFLOP_A / ms * 1e3 if (mode, T, h, w) == ("decode", 21, 64, 64) else None})
    print(json.dumps(res))
    if os.environ.get("OUT"):  # also append the result line to this JSON-lines file
        os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
        with open(os.environ["OUT"], "a") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
