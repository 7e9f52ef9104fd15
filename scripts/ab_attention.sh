#!/bin/bash
# A/B of the bf16 self-attention kernel: a base commit's library against the working tree's, alternated in one session.
#
#   scripts/ab_attention.sh build [REF]    no GPU needed.  Compiles REF's scail_b200/csrc (default HEAD~1, the parent of the
#                                          commit under test) into scail_b200/libscail_b200_base.so and rebuilds the product
#                                          library scail_b200/libscail_b200.so from the working tree.
#   scripts/ab_attention.sh run [ROUNDS]   one H100.  Prints the card's name, power limit and max SM clock, then ROUNDS times
#                                          (default 2) runs base and product in turn: scripts/perf_attn.py at N = 27 904 and
#                                          48 832 (b = 2, 40 heads), and bench.py --gpus 1 --no-extras --dump-outputs.  Ends
#                                          with the bench lines side by side and the latents of the two builds compared.
#
# SCAIL_LIB_VARIANT=base selects the base library; scail_b200._lib never rebuilds a variant, so the library `build` made is
# the one that runs.  Bench lines and latents go to $OUT (default: a new temporary directory, printed at the start).
set -euo pipefail
cd "$(dirname "$0")/.."

case "${1:-}" in
build)
    ref=${2:-HEAD~1}
    tmp=$(mktemp -d)
    trap 'rm -rf "$tmp"' EXIT
    git archive "$ref" scail_b200/csrc include | tar -x -C "$tmp"
    nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared -Xcompiler -fPIC \
        -o scail_b200/libscail_b200_base.so "$tmp/scail_b200/csrc/api.cu" -lcudart -ldl
    python -c "import sys; sys.path.insert(0, '.'); from scail_b200 import _lib; print(_lib.build(force=True))"
    echo "base = $(git rev-parse --short "$ref"): scail_b200/libscail_b200_base.so"
    ;;
run)
    rounds=${2:-2}
    test -f scail_b200/libscail_b200_base.so || { echo "no base library: run '$0 build' first" >&2; exit 1; }
    OUT=${OUT:-$(mktemp -d -t ab_attention.XXXXXX)}
    mkdir -p "$OUT"
    echo "results in $OUT"
    nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader -i 0
    for r in $(seq "$rounds"); do
        for v in base product; do
            var=""
            [ "$v" = base ] && var=base
            for n in 27904 48832; do
                echo -n "round $r $v perf_attn: "
                SCAIL_LIB_VARIANT=$var SDPA=0 N=$n python scripts/perf_attn.py
            done
            SCAIL_LIB_VARIANT=$var python bench.py --gpus 1 --no-extras --dump-outputs "$OUT/$v.$r" \
                > "$OUT/bench.$v.$r.json" 2> "$OUT/bench.$v.$r.err" || { tail -5 "$OUT/bench.$v.$r.err"; exit 1; }
        done
    done
    python - "$OUT" "$rounds" <<'EOF'
import json, os, sys
import numpy as np
out, rounds = sys.argv[1], int(sys.argv[2])
for r in range(1, rounds + 1):
    for v in ("base", "product"):
        line = [l for l in open(os.path.join(out, f"bench.{v}.{r}.json")) if l.startswith("{")][-1]
        b = json.loads(line)
        print(f"round {r} {v:8s} bench: {b['value']:.4f} steps/s, {b['ms_per_step']:.0f} ms/step, attention "
              f"{b['roofline']['avg_launch_ms']:.2f} ms/launch, share_of_step {b['roofline']['share_of_step']:.3f}")
for r in range(1, rounds + 1):
    xa = np.load(os.path.join(out, f"base.{r}", "x.npy"))
    xb = np.load(os.path.join(out, f"product.{r}", "x.npy"))
    rel = float(np.linalg.norm(xb.astype(np.float64) - xa) / np.linalg.norm(xa.astype(np.float64)))
    print(f"round {r} latent x.npy: bit-identical {np.array_equal(xa, xb)}, rel-L2 product vs base {rel:.3e}")
EOF
    ;;
*)
    echo "usage: $0 build [REF] | run [ROUNDS]" >&2
    exit 2
    ;;
esac
