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

/* In-place RMSNorm over D columns (fp32 math, affine weight) of 1 or 2 column slabs of a
 * [rows, ld] bf16 matrix, optionally followed by interleaved-pair RoPE with per-token fp32
 * tables cos/sin [rows_per_batch, 128].  Replaces RMSNorm.forward (dit_video_crossattn_sc_xc.py:61-68)
 * on q/k (:1070-1074, :1131-1142) and Rotary3DPositionEmbeddingMixin.attention_fn (:653-757). */
int scail_rmsnorm_rope(void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                       int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                       const float* cos, const float* sin, float eps, scail_stream_t stream);

/* Flash attention, head_dim 128, bf16, non-causal, softmax scale = scale.  Q/K/V are column slabs
 * (head h at columns [h*128, h*128+128)) of row-major matrices with leading dims ldq/ldk/ldv; batch b
 * starts at row b*q_batch_rows (Q, out) / b*kv_batch_rows (K, V); q_rows_total / kv_rows_total are the
 * allocated row counts (TMA bounds).  accumulate != 0 adds into out.
 * Replaces attention_fn_default -> F.scaled_dot_product_attention (sat/transformer_defaults.py:47-79). */
int scail_attention(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                    int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                    int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                    scail_stream_t stream);

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
int scail_cast_f32_bf16(const float* x, void* out, int64_t n, scail_stream_t stream);

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
