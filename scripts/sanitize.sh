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
# fp8 self-attention at small shapes: RMSNorm+RoPE fp8 form, V^T pre-pass (padding keys), attention_fp8 (partial last tile)
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck_fp8_attention.log" \
    python -m pytest tests/test_fp8_attention_gpu.py -q -x --timeout 600 \
    -k "rmsnorm_rope_fp8 and 1000 or rmsnorm_rope_fp8 and 130 or quant_vt and not 48832 or against_fp32_and_chain and not 27904 or small_model or refuses" \
    > "$OUT/memcheck_fp8_attention_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_fp8_attention_pytest.log"
tail -3 "$OUT/memcheck_fp8_attention_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck_fp8_attention.log" | head -5
# int8_qk self-attention at small shapes: RMSNorm+RoPE INT8 form, K smoothing and quantisation (ragged last chunk), the
# INT8 tile pooling, attention_int8qk dense and sparse (partial last tile)
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 99 --log-file "$OUT/memcheck_int8qk_attention.log" \
    python -m pytest tests/test_int8qk_attention_gpu.py -q -x --timeout 600 \
    -k "quantisers and 129 or quantisers and 1000 or dense and 1-2-129 or sparse_forms or tile_pool or small_model or abi" \
    > "$OUT/memcheck_int8qk_attention_pytest.log" 2>&1
echo "sanitizer exit code $?" >> "$OUT/memcheck_int8qk_attention_pytest.log"
tail -3 "$OUT/memcheck_int8qk_attention_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds" "$OUT/memcheck_int8qk_attention.log" | head -5
# adaptive tile selection at small shapes: tile pooling (bf16, e4m3 + scales, ragged last tile), device selection and
# compaction, and the per-(batch, head) sparse attention kernels; memcheck, then racecheck for the shared-memory selection
for tool in memcheck racecheck; do
    timeout 900 compute-sanitizer --tool $tool --error-exitcode 99 --log-file "$OUT/${tool}_adaptive.log" \
        python -m pytest tests/test_adaptive_attention_gpu.py -q -x --timeout 600 \
        -k "tile_pool and not 27904 or selection and 1000 or per_head and 1000 or mass_one_is and not 27904 or planted or refuses" \
        > "$OUT/${tool}_adaptive_pytest.log" 2>&1
    echo "sanitizer exit code $?" >> "$OUT/${tool}_adaptive_pytest.log"
    tail -3 "$OUT/${tool}_adaptive_pytest.log"; grep -E "ERROR SUMMARY|Invalid|out of bounds|hazard" "$OUT/${tool}_adaptive.log" | head -5
done
