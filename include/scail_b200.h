/* scail_b200 — C ABI of the Hopper-native (sm_90a) SCAIL denoising path (libscail_b200.so).
 *
 * Boundary contract (SURVEY.md §8b):
 *  - every buffer is caller-owned device memory (a PyTorch tensor's data_ptr); the library never
 *    frees or retains a pointer beyond the call (it caches TMA descriptors keyed on pointer+shape),
 *  - kernels are enqueued on the caller's stream, no implicit synchronisation,
 *  - every function returns 0 on success or a negative code; scail_last_error() returns a
 *    thread-local message.  Nothing here calls exit().
 *  - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 *
 * The reference (zai-org/SCAIL) has no native code on this path; each entry point names the
 * PyTorch call sites (reference file:line) whose work it replaces.  The ctypes precedent in the
 * reference is sat/quantization/kernels.py:70-121 (torch.empty outputs, c_void_p(data_ptr) args,
 * launch on torch.cuda.current_stream()).
 */
#ifndef SCAIL_B200_H
#define SCAIL_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* scail_stream_t; /* cudaStream_t */

const char* scail_last_error(void);
int scail_version(void);
/* device properties the host side sizes grids with; returns <0 when no CUDA device is usable */
int scail_device_sm_count(int device);

/* GEMM epilogues */
enum {
    SCAIL_EPI_BIAS = 0,
    SCAIL_EPI_BIAS_GELU = 1,      /* nn.GELU(approximate="tanh"), dit_video_crossattn_sc_xc.py:1296 */
    SCAIL_EPI_BIAS_GATE_RES = 2,  /* x + gate * (acc + bias),   dit_video_crossattn_sc_xc.py:1036,1050 */
    SCAIL_EPI_BIAS_RES = 3,       /* x + (acc + bias),          dit_video_crossattn_sc_xc.py:1042 */
    SCAIL_EPI_BIAS_SILU = 4,      /* nn.SiLU after linear,      dit_video_crossattn_sc_xc.py:1327-1331 */
    SCAIL_EPI_BIAS_GELU_ERF = 5   /* nn.GELU() in MLPProj,      dit_video_crossattn_sc_xc.py:38 */
};

/* C[M,N] = epilogue(A[M,K] @ W[N,K]^T); A, W, C bf16 row-major with leading dims lda/ldw/ldc
 * (elements, multiples of 8; ldc % 4 for a float32 C).  bias [N] bf16 or NULL; gate [B, gate_stride] bf16 indexed by
 * row / rows_per_batch; residual [M, ldr] bf16.  c_fp32 != 0 writes float32 C instead (not with the
 * residual epilogues: -1).  C, bias, gate and residual must be
 * 16-byte aligned (-1 otherwise).
 * Replaces ColumnParallelLinear.forward / RowParallelLinear.forward (sat/mpu/layers.py:230-243,
 * :425-444) and nn.Linear / nn.Conv3d-as-GEMM call sites of the DiT. */
int scail_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                    int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                    int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, scail_stream_t stream);

/* FP8 (e4m3) GEMM: C[M,N] = epilogue((A_q[M,K] @ W_q[N,K]^T) * scale_a[m] * scale_w[n]); the scaled fp32 product goes
 * through the same epilogues, in the same order, as scail_gemm_bf16.  A_q, W_q are e4m3 bytes (torch.float8_e4m3fn) with
 * leading dims lda/ldw in elements; K, lda, ldw must be multiples of 16.  scale_a [M] and scale_w [N] are float32 (one per
 * row, see scail_quant_rows_fp8).  C, bias, gate, residual as for scail_gemm_bf16; the output is bf16 only (c_fp32 != 0
 * is refused with -1). */
int scail_gemm_fp8(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                   int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                   int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                   const float* scale_w, scail_stream_t stream);

/* Row-wise e4m3 quantisation of a row-strided bf16 x [M, ldx]: scale[m] = amax(|x[m, :K]|) / 448 (IEEE division; 1 for an
 * all-zero row), q[m, k] = satfinite_rn(x[m, k] / scale[m]) written densely as e4m3 [M, K].  K % 16 == 0, K <= 16384,
 * ldx % 8 == 0; x and q 16-byte aligned. */
int scail_quant_rows_fp8(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream);

/* fp8_linear="int8": the linears' INT8 row format is the one of fp8_attention="int8_qk" (see scail_rmsnorm_rope_int8q),
 * one scale per row: scale[m] = amax(|x[m, :K]|) / 127 (IEEE division; 1 for an all-zero row), q[m, k] =
 * round-half-even(x[m, k] / scale[m]) saturated to [-127, 127].
 *
 * INT8 GEMM: C[M,N] = epilogue((float(A_q[M,K] @ W_q[N,K]^T) * scale_a[m]) * scale_w[n]).  The product is accumulated
 * exactly in s32 and converted once (round to nearest); then the same epilogues, in the same order, as scail_gemm_bf16.
 * A_q, W_q are int8 codes with leading dims lda/ldw in elements; K, lda, ldw must be multiples of 16 and K <= 131072
 * (K * 127^2 < 2^31).  Scales, C, bias, gate, residual and the bf16-only output as for scail_gemm_fp8. */
int scail_gemm_int8(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                    int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                    int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                    const float* scale_w, scail_stream_t stream);

/* Row-wise INT8 quantisation in the format above: x, q, scale and the limits as for scail_quant_rows_fp8, q int8 [M, K]. */
int scail_quant_rows_int8(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream);

/* out = modulate(LayerNorm(x)) per row.  gamma/beta (bf16 [D]) and shift/scale (bf16 [B, mod_stride])
 * are optional (NULL).  Reads rows [in_row_offset, in_row_offset+rows_out) of each batch of
 * in_batch_rows rows; writes [B*rows_out, D] densely.  D % 8 == 0, D <= 5120.
 * Replaces layer.input_layernorm / post_attention_layernorm / post_cross_attention_layernorm /
 * norm_final + modulate (dit_video_crossattn_sc_xc.py:1031-1032, 1039, 1045-1046, 825, 760-761). */
int scail_ln_modulate(const void* x, void* out, const void* gamma, const void* beta, const void* shift,
                      const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                      int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream);
/* The same rows quantised for scail_gemm_fp8: out_q e4m3 [B*rows_out, D] and out_scale float32 [B*rows_out], equal bit for
 * bit to scail_quant_rows_fp8 of what scail_ln_modulate writes.  D % 16 == 0. */
int scail_ln_modulate_fp8(const void* x, void* out_q, float* out_scale, const void* gamma, const void* beta, const void* shift,
                          const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                          int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream);
/* The same rows quantised for scail_gemm_int8: out_q int8 [B*rows_out, D], out_scale as for scail_ln_modulate_fp8, equal
 * bit for bit to scail_quant_rows_int8 of what scail_ln_modulate writes.  D % 16 == 0. */
int scail_ln_modulate_int8(const void* x, void* out_q, float* out_scale, const void* gamma, const void* beta, const void* shift,
                           const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                           int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream);

/* In-place RMSNorm over D columns (fp32 math, affine weight) of 1 or 2 column slabs of a
 * [rows, ld] bf16 matrix, optionally followed by interleaved-pair RoPE with per-token fp32
 * tables cos/sin [rows_per_batch, 128].  Replaces RMSNorm.forward (dit_video_crossattn_sc_xc.py:61-68)
 * on q/k (:1070-1074, :1131-1142) and Rotary3DPositionEmbeddingMixin.attention_fn (:653-757). */
int scail_rmsnorm_rope(void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                       int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                       const float* cos, const float* sin, float eps, scail_stream_t stream);
/* The same rows quantised for scail_attention_fp8 instead of written back: slab s goes to e4m3 rows q8_s [rows, ld8] with
 * one float32 scale per (token, head) in s8_s, head-major [B, D/128, L_pad] where B = rows / rows_per_batch and the
 * tokens [rows_per_batch, L_pad) are written as zeros.  Each 128-wide head of a token is one row of the e4m3 row format
 * (scail_quant_rows_fp8), equal bit for bit to quantising what scail_rmsnorm_rope writes.  buf is read only.
 * D % 128 == 0, ld8 % 16 == 0, rows_per_batch <= L_pad, L_pad % 128 == 0. */
int scail_rmsnorm_rope_fp8(const void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                           int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                           const float* cos, const float* sin, float eps, void* q8_0, float* s8_0, void* q8_1, float* s8_1,
                           int64_t ld8, int64_t L_pad, scail_stream_t stream);

/* V operand of scail_attention_fp8: V bf16 [B*L, H*head_dim] (column slab, leading dim ldv) -> vt e4m3 [B, H, 128, L_pad]
 * (keys contiguous; inside every 16-key group logical column k holds key 2*((k%16)/4) + (k%2) + 8*((k%4)/2); zeros past L)
 * and v_scale float32 [B, H, 128]: one e4m3 row-format scale per channel over the L keys.  amax_work: [B, H*128] 32-bit
 * workspace, zeroed and used by this call.  head_dim must be 128, L <= L_pad, L_pad % 128 == 0. */
int scail_quant_vt_fp8(const void* v, int64_t ldv, void* vt, float* v_scale, void* amax_work, int64_t B, int64_t H,
                       int64_t head_dim, int64_t L, int64_t L_pad, scail_stream_t stream);

/* FP8 (e4m3) self-attention, non-causal, softmax scale = scale, q_len == kv_len == L: Q, K e4m3 [B*L, H*128] with
 * leading dims ldq/ldk and scales q_scale/k_scale [B, H, L_pad] (scail_rmsnorm_rope_fp8); vt/v_scale from
 * scail_quant_vt_fp8.  out bf16 [B*L, ldo] (merged heads).  P = softmax numerator is quantised with the fixed scale 2^-8;
 * Hopper fp8 MMAs are accumulated per 128-key tile and summed in fp32.  head_dim must be 128. */
int scail_attention_fp8(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                        const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H, int64_t head_dim,
                        int64_t L, int64_t L_pad, float scale, scail_stream_t stream);
/* Block-sparse form of scail_attention_fp8 (see scail_attention_sparse for the map).  Extra checks: kv_tile_ptr and
 * kv_tile_idx non-NULL and 4-byte aligned, ceil(L/128) <= nnz <= ceil(L/128)^2. */
int scail_attention_fp8_sparse(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                               const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H,
                               int64_t head_dim, int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr,
                               const int32_t* kv_tile_idx, int64_t nnz, scail_stream_t stream);

/* Flash attention, head_dim 128, bf16, non-causal, softmax scale = scale.  Q/K/V are column slabs
 * (head h at columns [h*128, h*128+128)) of row-major matrices with leading dims ldq/ldk/ldv; batch b
 * starts at row b*q_batch_rows (Q, out) / b*kv_batch_rows (K, V); q_rows_total / kv_rows_total are the
 * allocated row counts (TMA bounds).  accumulate != 0 adds into out.
 * Replaces attention_fn_default -> F.scaled_dot_product_attention (sat/transformer_defaults.py:47-79). */
int scail_attention(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                    int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                    int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                    scail_stream_t stream);
/* Block-sparse self-attention (q_len == kv_len), same arguments and kernel as scail_attention plus a CSR map of 128 x 128
 * tiles shared by every (batch, head): query tile t (rows [128t, 128t + 128)) attends to exactly the keys of the key tiles
 * kv_tile_idx[kv_tile_ptr[t] .. kv_tile_ptr[t + 1]) (keys [128k, 128k + 128) clipped to kv_len); kv_tile_ptr int32
 * [ceil(q_len/128) + 1] from 0 to nnz, kv_tile_idx int32 [nnz].  Every row must be non-empty and strictly ascending with
 * indices < ceil(kv_len/128): the host checks only the pointers, their alignment and ceil(q_len/128) <= nnz <=
 * ceil(q_len/128) * ceil(kv_len/128); the contents are the caller's (scail_b200.ops.TileMap validates them). */
int scail_attention_sparse(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                           int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                           int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                           const int32_t* kv_tile_ptr, const int32_t* kv_tile_idx, int64_t nnz, scail_stream_t stream);

/* Per-(batch, head) block-sparse self-attention: as scail_attention_sparse, but (b, h) reads its own CSR map, kv_tile_ptr +
 * (b*H + h) * ptr_stride (ceil(L/128) + 1 entries from 0) and kv_tile_idx + (b*H + h) * idx_stride, with
 * ptr_stride >= ceil(L/128) + 1 and idx_stride >= ceil(L/128)^2 (the slot capacity).  No host nnz: the maps may be built on
 * the device (scail_attention_select_tiles), and their contents are trusted. */
int scail_attention_sparse_bh(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                              int64_t ldo, int64_t B, int64_t H, int64_t L, int64_t q_batch_rows, int64_t kv_batch_rows,
                              int64_t q_rows_total, int64_t kv_rows_total, float scale, const int32_t* kv_tile_ptr,
                              int64_t ptr_stride, const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream);
/* Per-(batch, head) form of scail_attention_fp8_sparse: the maps and strides as scail_attention_sparse_bh. */
int scail_attention_fp8_sparse_bh(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk,
                                  const float* k_scale, const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B,
                                  int64_t H, int64_t head_dim, int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr,
                                  int64_t ptr_stride, const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream);
/* fp8_attention="int8_qk": the INT8 row format is s = amax / 127 (IEEE division), q = round-half-even(x / s) saturated to
 * [-127, 127], s = 1 for an all-zero row; one row = one 128-wide head of one token.
 * RMSNorm(+RoPE) as scail_rmsnorm_rope over two slabs (nslabs must be 2): slab 0 (Q) goes to INT8 rows q8 [rows, ld8] with
 * scales q_scale head-major [B, D/128, L_pad] (zeros past rows_per_batch), equal bit for bit to quantising what
 * scail_rmsnorm_rope writes; slab 1 (K) is written back into buf in bf16 exactly as scail_rmsnorm_rope writes it.
 * D % 128 == 0, ld8 % 16 == 0, rows_per_batch <= L_pad, L_pad % 128 == 0. */
int scail_rmsnorm_rope_int8q(void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                             int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                             const float* cos, const float* sin, float eps, void* q8, float* q_scale, int64_t ld8, int64_t L_pad,
                             scail_stream_t stream);
/* Smoothed INT8 K: K bf16 [B*L, H*128] (column slab, leading dim ldk) -> kbar float32 [B, H*128], the mean over the L keys
 * of each batch element (summed in fp64 over fixed 256-key chunks, chunks added in ascending order, divided by L in fp64,
 * rounded once to fp32), and K' = f32(k) - kbar (one fp32 rounding) in the INT8 row format: k8 [B*L, ld8], k_scale
 * [B, H, L_pad] with zeros past L.  partial: fp64 workspace of partial_len >= B*ceil(L/256)*H*128 entries.
 * Three launches, no atomics and no host reads: bit-reproducible and capturable in a CUDA graph.  L <= L_pad, L_pad % 128 == 0,
 * H*128 <= 5120. */
int scail_quant_k_int8(const void* k, int64_t ldk, void* k8, int64_t ld8, float* k_scale, float* kbar, double* partial,
                       int64_t partial_len, int64_t B, int64_t H, int64_t L, int64_t L_pad, scail_stream_t stream);
/* Self-attention with INT8 Q and K (scail_rmsnorm_rope_int8q, scail_quant_k_int8) and the e4m3 V^T of scail_quant_vt_fp8:
 * S = Q K^T in exact s32, then as scail_attention_fp8.  kv_tile_ptr NULL: dense.  Otherwise a block-sparse map as
 * scail_attention_sparse_bh with ptr_stride / idx_stride per (batch, head), or both 0 for one map shared by every (batch,
 * head); its contents are trusted (the host checks pointers, alignment and strides). */
int scail_attention_int8qk(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                           const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H, int64_t head_dim,
                           int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr, int64_t ptr_stride,
                           const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream);
/* Tile pooling for adaptive tile selection: out fp32 [B, H, ceil(L/128), 128] = the mean over each 128-row tile's valid rows
 * of one self-attention operand, x [B*L, ldx] with head h at columns [h*128, h*128+128).  fp8 == 0: x is bf16 and x_scale
 * NULL.  fp8 == 1: x is e4m3 and the value is x * x_scale[b, h, row] with x_scale fp32 [B, H, L_pad]
 * (scail_rmsnorm_rope_fp8).  Summed in ascending row order in fp64: bit-reproducible. */
int scail_attention_tile_pool(const void* x, int64_t ldx, const float* x_scale, int fp8, float* out, int64_t B, int64_t H,
                              int64_t L, int64_t L_pad, scail_stream_t stream);
/* scail_attention_tile_pool of an INT8 operand (fp8_attention="int8_qk": scail_rmsnorm_rope_int8q, scail_quant_k_int8): the
 * value is x * x_scale[b, h, row], x int8 [B*L, ldx], x_scale fp32 [B, H, L_pad].  Pooling the smoothed K' instead of K
 * shifts every s_k of one query tile by the same amount, so the selection does not change. */
int scail_attention_tile_pool_int8(const void* x, int64_t ldx, const float* x_scale, float* out, int64_t B, int64_t H, int64_t L,
                                   int64_t L_pad, scail_stream_t stream);
/* Adaptive tile selection on the device.  qbar, kbar fp32 [B, H, n, 128] (scail_attention_tile_pool), n = ceil(L/128).
 * Query tile q of (b, h) lists the key tiles with e_k = n_k exp(s_k - max s), s_k = qbar_q . kbar_k / sqrt(128), n_k the
 * valid keys of tile k: always k == q and every k < ceil(n_ref/128) (reference tokens), then the others by e_k descending
 * (ties: lower k) until the listed sum reaches mass * sum_k e_k or max_tiles were taken that way (max_tiles < 0: no cap).
 * mass >= 1 takes every tile (up to the cap); mass == 0 only the forced ones.  Writes the per-(b, h) maps of
 * scail_attention_sparse_bh (rows ascending).  scratch: int32, at least B*H*n*(1 + ceil(n/32)) entries (scratch_len).
 * n <= 2048.  No host synchronisation: the selection can be captured in a CUDA graph. */
int scail_attention_select_tiles(const float* qbar, const float* kbar, int64_t B, int64_t H, int64_t L, int64_t n_ref, double mass,
                                 int64_t max_tiles, int32_t* kv_tile_ptr, int64_t ptr_stride, int32_t* kv_tile_idx,
                                 int64_t idx_stride, int32_t* scratch, int64_t scratch_len, scail_stream_t stream);

/* Context parallelism: attention over a SUBSET of the keys, to be merged later.  Keys are the rows
 * [kv_off0, kv_off0 + kv_len0) and (optionally, kv_len1 > 0) [kv_off1, kv_off1 + kv_len1) of every batch of kv_batch_rows rows
 * ("every shard but mine").  Writes the partial result normalised by its own row sum as float32 o32 [rows, ldo32] and
 * state [rows * H] = (running max in log2 units, row sum) float2.  Same kernel as scail_attention.
 * Replaces the all_to_all_4D + SDPA + all_to_all_4D sequence of UlyssesAttention.forward (sat/mpu/ulysses_attn_layer.py:41-110)
 * together with scail_attention_merge. */
int scail_attention_partial(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, float* o32,
                            int64_t ldo32, void* state, int64_t B, int64_t H, int64_t q_len, int64_t kv_off0, int64_t kv_len0,
                            int64_t kv_off1, int64_t kv_len1, int64_t q_batch_rows, int64_t kv_batch_rows, int64_t q_rows_total,
                            int64_t kv_rows_total, float scale, scail_stream_t stream);
/* out (bf16 [rows, ldo], head h at columns h*128..) = softmax-consistent combination of two partial results over disjoint key
 * sets: (w_a O_a + w_b O_b) / (w_a + w_b), w_x = l_x 2^(m_x - max(m_a, m_b)). */
int scail_attention_merge(const float* o32_a, const void* state_a, const float* o32_b, const void* state_b, void* out,
                          int64_t ldo32, int64_t ldo, int64_t rows, int64_t H, scail_stream_t stream);

/* Context-parallel collective (the path's one exchange step: the per-block K/V all-gather over the sequence-parallel group,
 * replacing the 12 all_to_all_single calls per block of sat/mpu/ulysses_attn_layer.py:41-110 / sat/mpu/all_to_all.py:15-109).
 * NCCL is bound at run time (dlopen of libnccl.so.2; `nccl_path` may name a specific file, NULL = the one already loaded by the
 * process).  scail_cp_unique_id: 128-byte id created on one rank and shipped to the others by the host (e.g. a
 * torch.distributed broadcast).  scail_cp_init: join with the CURRENT CUDA device, returns a handle >= 0.
 * scail_cp_allgather: recv = nranks consecutive slots of bytes_per_rank bytes, rank r's data in slot r (send may alias it);
 * enqueued on the group's own high-priority stream after everything already on compute_stream (event hand-off), returns at
 * once.  scail_cp_wait: compute_stream waits (device-side) for the group's outstanding collectives. */
int scail_cp_unique_id(void* out128, const char* nccl_path);
int scail_cp_init(const void* unique_id128, int rank, int nranks, const char* nccl_path);
int scail_cp_allgather(int handle, const void* send, void* recv, int64_t bytes_per_rank, scail_stream_t compute_stream);
int scail_cp_wait(int handle, scail_stream_t compute_stream);
int scail_cp_destroy(int handle);

/* mod[b, i] = emb[b, i] + param[i]  (shared-AdaLN modulation vectors, dit_video_crossattn_sc_xc.py:1025-1028, 823) */
int scail_adaln_modulation(const void* emb, const void* param, void* out, int64_t B, int64_t n, scail_stream_t stream);
int scail_silu(const void* x, void* out, int64_t n, scail_stream_t stream);
/* timestep_embedding (sgm/modules/diffusionmodules/util.py:207-231): t fp32 [B] -> bf16 [B, dim] (cos||sin) */
int scail_timestep_embedding(const float* t, void* out, int64_t B, int64_t dim, scail_stream_t stream);

/* Patch gather for ImagePatchEmbeddingMixin (dit_video_crossattn_sc_xc.py:99-130) including the mask
 * channels appended by DiffusionTransformer.forward (:1468-1503) when cin == 16 (x: zeros, ref/pose: ones);
 * cin == 20 reads them from the inputs.  x [B,T,cin,H,W], ref [Br,1,cin,H,W], pose [Bp,T,cin,H/2,W/2] bf16
 * -> a_main [B,(1+T)*H/2*W/2, 80], a_pose [B, T*H/4*W/4, 80] bf16 (feature order c*4 + p*2 + q). */
int scail_patchify(const void* x, const void* ref, const void* pose, void* a_main, void* a_pose, int64_t B,
                   int64_t Br, int64_t Bp, int64_t T, int64_t H, int64_t W, int64_t cin, scail_stream_t stream);
/* unpatchify (dit_video_crossattn_sc_xc.py:764-784): lin [B, T*Hp*Wp, 64] -> out [B, T, 16, 2Hp, 2Wp], bf16 */
int scail_unpatchify(const void* lin, void* out, int64_t B, int64_t T, int64_t Hp, int64_t Wp, scail_stream_t stream);
/* x (fp32, n elements) += dsigma * (v_u + scale*(v_c - v_u)), v bf16 [2, n]
 * (guiders.py:41-45, sampling_utils.py:7-10, sampling.py:960-963) */
int scail_cfg_euler(float* x, const void* v, int64_t n, float scale, float dsigma, scail_stream_t stream);
/* One UniPC solver step (scail_b200/unipc.py), in place, one pass over n fp32 elements (n % 4 == 0).  v is the bf16 CFG
 * pair [2, n] as scail_cfg_euler reads it; slots holds n_slots (1..3) fp32 model outputs of n elements, slot s at
 * slots + s * slot_stride floats (slot_stride >= n, a multiple of 4); x, x_last, v and slots are 16-byte aligned.
 * coef is a host array of 10 floats {a_x, a_0, a_1, a_2, a_m, b_y, b_0, b_1, b_2, b_m}, passed to the kernel by value;
 * the coefficients of slots >= n_slots must be 0.  Per element, each product and sum rounded separately (no FMA):
 * g = u + scale*(c - u); m = x - sigma*g; y = a_x*x_last + a_s*M_s (slot order) + a_m*m if correct, else y = x;
 * z = b_y*y + b_s*M_s (slot order) + b_m*m; then x = z, x_last = y, slot write_slot = m.  A slot whose coefficients are 0
 * is neither read nor added; all reads precede the writes, so write_slot may be a slot the step reads. */
int scail_unipc_step(float* x, float* x_last, const void* v, float* slots, int64_t slot_stride, int64_t n_slots,
                     int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                     scail_stream_t stream);
int scail_cast_f32_bf16(const float* x, void* out, int64_t n, scail_stream_t stream);
/* CFG cache (scail_b200/cfg_cache.py).  n fp32 elements (n % 4 == 0); every pointer below is 16-byte aligned except
 * partials (4) and out (8).
 * scail_cfg_cache_delta: from the bf16 CFG pair v [2, n] (as scail_cfg_euler reads it), d_new = f32(c) - f32(u) (one
 * subtraction, rounded once) and out = {sum |d_new - d_ref|, sum |d_ref|, ratio, 0} (fp64; ratio = +inf when the
 * denominator is 0).  fp32 partial sums per CTA over a fixed partition of the elements (partials: at least 2 * 1024
 * floats), then one CTA adds them in fp64 in a fixed order: bit-reproducible, no floating-point atomics.  Two launches.
 * scail_cfg_euler_cached: the conditional-only Euler step from c, bf16 [n], and delta: per element, each product and sum
 * rounded separately (no FMA), u = c - delta; g = u + scale*(c - u); x = x + dsigma*g.
 * scail_unipc_step_cached: scail_unipc_step with u = f32(c) - delta in place of the pair's u (c bf16 [n], delta fp32 [n]);
 * the same checks and every later instruction shared, so where delta = f32(c) - f32(u) is exact the two agree bit for
 * bit. */
int scail_cfg_cache_delta(const void* v, const float* d_ref, float* d_new, float* partials, int64_t partials_len, double* out,
                          int64_t n, scail_stream_t stream);
int scail_cfg_euler_cached(float* x, const void* c, const float* delta, int64_t n, float scale, float dsigma,
                           scail_stream_t stream);
int scail_unipc_step_cached(float* x, float* x_last, const void* c, const float* delta, float* slots, int64_t slot_stride,
                            int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma, int correct,
                            const float* coef, scail_stream_t stream);
/* CFG cache forecast (CFGCache(order >= 1)): n_slots (1..3) fp32 delta slots of n elements, slot s at slots + s*slot_stride
 * floats (slot_stride >= n, a multiple of 4), and coef: 3 host floats, the forecast coefficient of each slot (0 for every
 * slot s >= n_slots).  The forecast is t = c0*S0, then t = t + c1*S1, then t = t + c2*S2, each product and sum rounded on
 * its own (no FMA); a slot whose coefficient is exactly 0 is not read, and with no active slot t = 0.
 * scail_cfg_cache_delta_forecast: slot write_slot = f32(c) - f32(u) from the pair v [2, n] and out = {sum |d_new - t|,
 * sum |t|, ratio, 0}, in scail_cfg_cache_delta's partition and order (bit-reproducible; with coef = 1 on one slot alone
 * its sums are scail_cfg_cache_delta's with d_ref = that slot, bit for bit).  The write slot may be one t reads.
 * scail_cfg_euler_cached_forecast: scail_cfg_euler_cached with delta = t.
 * scail_unipc_step_cached_forecast: scail_unipc_step_cached with delta = t of the delta slots (dslots, dslot_stride,
 * n_dslots, dcoef); the UniPC slots and coefficients as scail_unipc_step. */
int scail_cfg_cache_delta_forecast(const void* v, float* slots, int64_t slot_stride, int64_t n_slots, int64_t write_slot,
                                   const float* coef, float* partials, int64_t partials_len, double* out, int64_t n,
                                   scail_stream_t stream);
int scail_cfg_euler_cached_forecast(float* x, const void* c, const float* slots, int64_t slot_stride, int64_t n_slots,
                                    const float* coef, int64_t n, float scale, float dsigma, scail_stream_t stream);
int scail_unipc_step_cached_forecast(float* x, float* x_last, const void* c, const float* dslots, int64_t dslot_stride,
                                     int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride, int64_t n_slots,
                                     int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                                     scail_stream_t stream);
/* CFG-Zero* guidance (scail_b200/guidance.py).  n fp32 elements (n % 4 == 0); every tensor pointer is 16-byte aligned
 * except partials (4), out (8) and u_scale (4), a single fp32 value in device memory.
 * scail_cfg_zero_scale: s* = <c, u> / (|u|^2 + 1e-8) over all n elements, with u and c by `form`:
 *   0: v is the bf16 CFG pair [2, n]; delta, delta_stride, n_dslots and dcoef are not read;
 *   1: v is c alone, bf16 [n], and u = f32(c) - delta, delta fp32 [n]; delta_stride, n_dslots and dcoef are not read;
 *   2: v is c alone and u = f32(c) - t, t the forecast of the delta slots (delta, delta_stride, n_dslots, dcoef) as in
 *      scail_cfg_euler_cached_forecast.
 * u is formed as the update of the same form forms it.  fp32 partial sums of c*u and u*u per CTA over a fixed partition
 * (each product and sum rounded on its own; partials: at least 2 * 1024 floats), then one CTA adds them in fp64 in a fixed
 * order: out = {dot, norm, 0, 0} (fp64) and *u_scale = dot / (norm + 1e-8) in fp64, rounded once to fp32.
 * Bit-reproducible; two launches.
 * The scaled twins take one more argument, u_scale, and form u' = (*u_scale) * u (one rounded product) where their
 * unscaled form uses u:
 *   scail_cfg_euler_scaled: per element, each product and sum rounded on its own, u' = s*u; g = u' + scale*(c - u');
 *     x = x + dsigma*g (v the pair [2, n]; x and v 16-byte aligned).  Not bit-equal to scail_cfg_euler at s = 1, whose
 *     arithmetic the compiler may contract.
 *   scail_cfg_euler_cached_scaled, scail_cfg_euler_cached_forecast_scaled, scail_unipc_step_scaled,
 *   scail_unipc_step_cached_scaled, scail_unipc_step_cached_forecast_scaled: every other instruction and check as in the
 *     unscaled entry point, so *u_scale == 1 gives its result bit for bit. */
int scail_cfg_zero_scale(int form, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots, const float* dcoef,
                         float* partials, int64_t partials_len, double* out, float* u_scale, int64_t n, scail_stream_t stream);
int scail_cfg_euler_scaled(float* x, const void* v, int64_t n, float scale, float dsigma, const float* u_scale,
                           scail_stream_t stream);
int scail_cfg_euler_cached_scaled(float* x, const void* c, const float* delta, int64_t n, float scale, float dsigma,
                                  const float* u_scale, scail_stream_t stream);
int scail_cfg_euler_cached_forecast_scaled(float* x, const void* c, const float* slots, int64_t slot_stride, int64_t n_slots,
                                           const float* coef, int64_t n, float scale, float dsigma, const float* u_scale,
                                           scail_stream_t stream);
int scail_unipc_step_scaled(float* x, float* x_last, const void* v, float* slots, int64_t slot_stride, int64_t n_slots,
                            int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                            const float* u_scale, scail_stream_t stream);
int scail_unipc_step_cached_scaled(float* x, float* x_last, const void* c, const float* delta, float* slots,
                                   int64_t slot_stride, int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma,
                                   int correct, const float* coef, const float* u_scale, scail_stream_t stream);
int scail_unipc_step_cached_forecast_scaled(float* x, float* x_last, const void* c, const float* dslots, int64_t dslot_stride,
                                            int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride,
                                            int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma,
                                            int correct, const float* coef, const float* u_scale, scail_stream_t stream);
/* APG, adaptive projected guidance (scail_b200/guidance.py).  The fp32 latent x holds n elements in `frames` frames of
 * n / frames elements (n % (4 * frames) == 0, 1 <= frames <= 65535); u and c come by `form` as in scail_cfg_zero_scale
 * (0: the pair [2, n]; 1: c alone with u = f32(c) - delta; 2: c alone with u = f32(c) - the forecast of the delta slots).
 * x, v, delta, avg and m are 16-byte aligned, partials 4-byte, sums and factors 8-byte.  Per element, each product and sum
 * rounded on its own: D_c = x - sigma*c, diff = D_c - (x - sigma*u).
 * scail_apg_reduce (pass 1): with avg (fp32 [n], may be null) avg = diff + momentum*avg, read and written once, and diff =
 *   avg.  fp32 partial sums of diff*diff, diff*D_c and D_c*D_c per (frame, CTA) over a partition fixed by the shape
 *   (partials: at least 3 * frames * 32 floats).  Bit-reproducible.
 * scail_apg_finish (pass 2): per frame, the partials added in fp64 in a fixed order -> sums [frames, 4] fp64 = {|diff|^2,
 *   <diff, D_c>, |D_c|^2, 0} and factors [frames, 2] = {f, p}, each computed in fp64 and rounded once to fp32: f =
 *   norm_threshold / |diff| if norm_threshold > 0 and |diff| > norm_threshold, else 1; p = f <diff, D_c> / |D_c|^2, 0 when
 *   |D_c|^2 = 0.
 * scail_apg_update: diff as pass 1 left it (avg when given, which then must be the average pass 1 wrote; else formed again
 *   by the same instructions); par = p*D_c; orth = f*diff - par; D_g = D_c + wm1*(orth + eta*par).  With m (fp32 [n]) D_g
 *   -> m and x is only read; with m null, x = x + k_euler*(x - D_g) in place.
 * scail_unipc_step_dpred: scail_unipc_step with the data prediction m read from `m` (fp32 [n]) in place of x - sigma*g;
 *   every other instruction and check as there. */
int scail_apg_reduce(int form, const float* x, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots,
                     const float* dcoef, float* avg, float sigma, float momentum, float* partials, int64_t partials_len,
                     int64_t frames, int64_t n, scail_stream_t stream);
int scail_apg_finish(const float* partials, int64_t partials_len, double* sums, float* factors, double norm_threshold,
                     int64_t frames, int64_t n, scail_stream_t stream);
int scail_apg_update(int form, float* x, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots,
                     const float* dcoef, const float* avg, const float* factors, float* m, float sigma, float wm1, float eta,
                     float k_euler, int64_t frames, int64_t n, scail_stream_t stream);
int scail_unipc_step_dpred(float* x, float* x_last, const float* m, float* slots, int64_t slot_stride, int64_t n_slots,
                           int64_t write_slot, int64_t n, int correct, const float* coef, scail_stream_t stream);

/* First-block residual cache (scail_b200/step_cache.py).  Token tensors are bf16 [B, N, d] (ref || noise || pose rows of
 * each batch element); the noise rows are rows [n_ref, n_ref + n_seq) of each element.  d % 8 == 0, B*N*d/8 < 2^31, and
 * every bf16/fp32 tensor is contiguous and 16-byte aligned.
 * scail_step_cache_indicator: r = bf16_rn(f32(h1) - f32(h0)) -> r_new, the noise rows of h1 -> h1c [B, n_seq, d], and
 * out = {sum |r - r_ref|, sum |r_ref|, ratio, 0} (fp64; ratio = +inf when the denominator is 0).  fp32 partial sums per CTA
 * over a fixed partition of the elements (partials: at least 2 * 1024 floats), then one CTA adds them in fp64 in a fixed
 * order: bit-reproducible, no floating-point atomics.  Two launches.
 * scail_step_cache_update: R [B, n_seq, d] fp32 = f32(h[noise rows]) - f32(h1c).
 * scail_step_cache_apply: in place on the noise rows of h, h = bf16_rn(f32(h) + R). */
int scail_step_cache_indicator(const void* h0, const void* h1, const void* r_ref, void* r_new, void* h1c, float* partials,
                               int64_t partials_len, double* out, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                               scail_stream_t stream);
int scail_step_cache_update(const void* h, const void* h1c, float* R, int64_t B, int64_t N, int64_t d, int64_t n_ref,
                            int64_t n_seq, scail_stream_t stream);
int scail_step_cache_apply(void* h, const float* R, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                           scail_stream_t stream);
/* Taylor forecast of the skipped blocks' residual (FirstBlockCache(order >= 1)).  R_slots holds n_slots (1..3) fp32
 * [B, n_seq, d] slots, slot s at R_slots + s * slot_stride floats (slot_stride >= B*n_seq*d, a multiple of 4).  The slot
 * index and the coefficients are read from device memory when the kernel runs, so one captured graph serves every step.
 * scail_step_cache_update_slot: R_slots[*slot] = f32(h[noise rows]) - f32(h1c); a *slot outside [0, n_slots) writes nothing.
 * scail_step_cache_apply_forecast: in place on the noise rows of h, t = c0*R0, t = t + c1*R1, t = t + c2*R2 (slot order,
 * each product and sum rounded separately), then h = bf16_rn(f32(h) + t).  A slot with coef[s] == 0 is neither read nor
 * added; with every coefficient 0, h is left unchanged. */
int scail_step_cache_update_slot(const void* h, const void* h1c, float* R_slots, int64_t slot_stride, int64_t n_slots,
                                 const int* slot, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                                 scail_stream_t stream);
int scail_step_cache_apply_forecast(void* h, const float* R_slots, int64_t slot_stride, int64_t n_slots, const float* coef,
                                    int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq, scail_stream_t stream);

/* ---- Wan2.1 VAE decode (sgm/models/wan_vae.py); activations channels-last bf16 [T, H, W, C] ---- */
enum { SCAIL_CONV_EPI_BIAS = 0, SCAIL_CONV_EPI_BIAS_RES = 1, SCAIL_CONV_EPI_HEAD_CLAMP = 2 };

/* Causal 3-D convolution as an implicit GEMM on wgmma (CausalConv3d.forward, wan_vae.py:17-36; also the
 * per-frame Conv2d 3x3 of Resample with KT = 1, :77-83).  x [T,H,W,Cin]; w2 = weight repacked to
 * [Cout, KT*KH*KW*Cin] (tap-major, channel-minor); stride 1, "same" spatial zero padding, causal temporal
 * padding (KT-1 zero frames on the left).  Output column c is written to frame t*fmul + c/ocols, channel
 * c%ocols of out [*, H, W, ldo] (fmul=2, ocols=Cout/2 interleaves time_conv's channel halves as frames,
 * wan_vae.py:134-137).  epilogue: +bias | +bias+residual [T,H,W,ldr] (ResidualBlock, :220) |
 * head: +bias, clamp(-1,1), fp32 planes [Cout, T, H, W] (:421, :662-664).
 * norm_gamma/out2 (optional, Cout == 96, 3x3 taps, W >= 128): additionally write out2 [T,H,W,96] =
 * SiLU(RMS_norm(value) * gamma), the input of the NEXT conv (ResidualBlock.residual[0..1] / [3..4], :194-198);
 * out may then be NULL when the raw value is not needed. */
int scail_conv3d_cl(const void* x, int64_t T, int64_t H, int64_t W, int64_t Cin, const void* w2, int64_t Cout, int KT,
                    int KH, int KW, const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                    int64_t ocols, int fmul, int epilogue, const void* norm_gamma, void* out2, scail_stream_t stream);
/* Strided variant for the encoder's Resample (wan_vae.py:87-96, 143-159): x [T_in,H_in,W_in,Cin] -> out [T_out,H_out,W_out,ldo];
 * tap (dt,dh,dw) of output (t,h,w) reads input (t*tstride + dt + toff, h*sstride + dh - pad_h, w*sstride + dw - pad_w),
 * out-of-range inputs are zero.  downsample2d/3d spatial conv: sstride 2, pads 0 (ZeroPad2d((0,1,0,1)));
 * downsample3d time_conv: 3x1x1, tstride 2, toff 0 on frames 1.. (frame 0 bypasses it). */
int scail_conv3d_strided_cl(const void* x, int64_t T_in, int64_t H_in, int64_t W_in, int64_t Cin, const void* w2, int64_t Cout,
                            int KT, int KH, int KW, const void* bias, void* out, int64_t ldo, int64_t T_out, int64_t H_out,
                            int64_t W_out, int sstride, int pad_h, int pad_w, int tstride, int toff, scail_stream_t stream);

/* Temporally chunked VAE runs (CausalConv3d.forward(x, cache_x), wan_vae.py:28-36): the same convolutions with a causal
 * HISTORY, hist [T_hist, H, W, Cin] bf16 channels-last (same H, W, Cin as x; for the strided call the input extent
 * H_in, W_in), holding the frames that precede x[0] in the conv's input stream.  A tap whose input frame
 * ct = t*tstride + dt + toff is < 0 reads hist frame ct + T_hist; when that is still < 0 it reads zeros (so a 1-frame
 * history means "one real frame, then zero padding").  0 <= T_hist <= KT-1; T_hist == 0 ignores hist (may be NULL) and
 * is exactly scail_conv3d_cl / scail_conv3d_strided_cl, which forward here.  hist must be 16-byte aligned (C % 8 == 0).
 * The taps, channel slices and their summation order do not depend on where a frame comes from, so a conv over
 * cat(hist, x) and this call agree bit for bit on the frames of x.
 * Head epilogue only: out_plane_stride (elements per output channel plane; 0 = T*H*W) and out_frame_offset place the
 * T output frames at frames [out_frame_offset, out_frame_offset + T) of a larger fp32 [Cout, T_total, H, W] output
 * (out_plane_stride = T_total*H*W); both must be 0 for the bf16 epilogues.
 * Strided variant: the downsample3d time_conv of a later chunk is tstride 2, toff -1 with the last input frame of the
 * previous chunk as a 1-frame history (the reference's x[:, :, -1:] cache, wan_vae.py:151-157). */
int scail_conv3d_cl_hist(const void* x, int64_t T, int64_t H, int64_t W, int64_t Cin, const void* w2, int64_t Cout, int KT,
                         int KH, int KW, const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                         int64_t ocols, int fmul, int epilogue, const void* norm_gamma, void* out2, const void* hist,
                         int64_t T_hist, int64_t out_plane_stride, int64_t out_frame_offset, scail_stream_t stream);
int scail_conv3d_strided_cl_hist(const void* x, int64_t T_in, int64_t H_in, int64_t W_in, int64_t Cin, const void* w2,
                                 int64_t Cout, int KT, int KH, int KW, const void* bias, void* out, int64_t ldo, int64_t T_out,
                                 int64_t H_out, int64_t W_out, int sstride, int pad_h, int pad_w, int tstride, int toff,
                                 const void* hist, int64_t T_hist, scail_stream_t stream);
/* RMS_norm over channels (F.normalize * sqrt(C) * gamma, wan_vae.py:39-54), optional SiLU; [npix, C] bf16 */
int scail_rmsnorm_cl(const void* x, const void* gamma, void* out, int64_t npix, int64_t C, int silu, scail_stream_t stream);
/* nearest-exact 2x spatial upsample (wan_vae.py:57-63): [frames,H,W,C] -> [frames,2H,2W,C] */
int scail_upsample2x_cl(const void* x, void* out, int64_t frames, int64_t H, int64_t W, int64_t C, scail_stream_t stream);
/* z [16,T,h,w] bf16 -> z / inv_std + mean, channels-last [T,h,w,16] (WanVAE_.decode, wan_vae.py:547-551) */
int scail_vae_latent_to_cl(const void* z, const float* mean, const float* inv_std, void* out, int64_t T, int64_t h,
                           int64_t w, scail_stream_t stream);
/* p = softmax(s * scale) per row; s fp32 [rows, cols] -> p bf16 (mid-block attention, wan_vae.py:252-256) */
int scail_softmax_rows(const float* s, void* p, int64_t rows, int64_t cols, float scale, scail_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
