#!/bin/bash
# compute-sanitizer memcheck over the small-shape kernel tests (SURVEY §5: the reference has no sanitizer runs).
# Logs go to $SANITIZE_OUT (default: sanitize_logs/, ignored by git).
OUT=${SANITIZE_OUT:-sanitize_logs}
mkdir -p "$OUT"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck.log" \
    python -m pytest tests/test_kernels_gpu.py -q -x --timeout 600 \
    -k "gemm_bias and 128-256-64 or gemm_epilogues or ln_modulate and 256 or rmsnorm_rope and 256 or test_attention and 1-2-256-256 or test_attention and 300 or small_ops or patchify or gemm_cta_pair and 2048 or attention_partial and 4-200" \
    > "$OUT/memcheck_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_pytest.log"
tail -3 "$OUT/memcheck_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck.log" | head -5
# conv kernels with a causal history (chunked VAE): history map, strided time_conv, head frame offset
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck_chunked.log" \
    python -m pytest tests/test_vae_chunked_gpu.py -q -x --timeout 600 -k "history or head_writes" \
    > "$OUT/memcheck_chunked_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_chunked_pytest.log"
tail -3 "$OUT/memcheck_chunked_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck_chunked.log" | head -5
# GEMM staged epilogue at small shapes: TMA residual loads and clipped TMA stores at ragged M / N and column slabs
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck_gemm_tiles.log" \
    python -m pytest tests/test_gemm_tiles_gpu.py -q -x --timeout 600 -k "not bench_shapes" \
    > "$OUT/memcheck_gemm_tiles_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_gemm_tiles_pytest.log"
tail -3 "$OUT/memcheck_gemm_tiles_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck_gemm_tiles.log" | head -5
# fp8 linears at small shapes: row quantiser, fp8 LayerNorm, fp8 GEMM (ragged tiles, gate rows, column slabs)
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck_fp8.log" \
    python -m pytest tests/test_fp8_gpu.py -q -x --timeout 600 -k "ragged or gate_rows or column_slabs or refuses or small_model" \
    > "$OUT/memcheck_fp8_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_fp8_pytest.log"
tail -3 "$OUT/memcheck_fp8_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck_fp8.log" | head -5
