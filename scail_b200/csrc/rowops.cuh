// HBM-bound row / elementwise kernels of the SCAIL DiT step (everything that is not a GEMM or attention).
// One warp per row, 16-byte vectorised loads, fp32 statistics, bf16 in/out.
#pragma once
#include <cuda_fp8.h>

#include "sm90.cuh"

namespace scail {

// Row kernels: ONE 128-thread block per row, each thread holds <= ROW_MAXV 16-byte vectors (D <= 5120, D % 8 == 0).
// Round 1 used a warp per row (20 vectors = 80+ data registers per lane -> 194 registers, one 8-warp block per SM whose
// warps load, reduce and store in lockstep, so reads and writes never overlapped: 0.44-0.46 of HBM peak).  With ~48
// registers per thread, 16 rows are resident per SM at independent phases, which is what keeps HBM busy in both directions.
constexpr int ROW_THREADS = 128;
constexpr int ROW_MAXV = 5;  // vectors per thread: 5 * 128 * 8 = 5120 columns

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// sum over the 128-thread block; `red` is a 4-float shared scratch (one slot per warp), safe to reuse after the call returns
__device__ __forceinline__ float row_block_sum(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    const float t = (red[0] + red[1]) + (red[2] + red[3]);
    __syncthreads();
    return t;
}

// max over the 128-thread block; same contract as row_block_sum
__device__ __forceinline__ float row_block_max(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    const float t = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    return t;
}

// ---- e4m3 row quantisation, the one format of the fp8 GEMMs: s = amax(|row|) / 448 (IEEE division), q = satfinite_rn(x / s);
// an all-zero row gets s = 1 and q = 0.  torch: (x.float() / s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)
constexpr float FP8_E4M3_MAX = 448.0f;

__device__ __forceinline__ float absmax_bf16x2(float m, uint32_t w) {
    const float2 f = unpack_bf16(w);
    return fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
}
__device__ __forceinline__ float fp8_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, FP8_E4M3_MAX) : 1.0f; }
// 8 bf16 -> 8 e4m3 bytes
__device__ __forceinline__ uint2 quant_bf16x8(const uint4 v, float s) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t h[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(w[k]);
        h[k] = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f.x, s), __fdiv_rn(f.y, s)), __NV_SATFINITE, __NV_E4M3);
    }
    return make_uint2(h[0] | (h[1] << 16), h[2] | (h[3] << 16));
}

// One 128-thread block per row of a row-strided bf16 [M, K] (K % 16 == 0, K <= 8 * ROW_THREADS * V): the row stays in registers
// between the amax reduction and the quantisation, so it is read once.
template <int V>
__global__ void __launch_bounds__(ROW_THREADS) quant_rows_fp8_kernel(const __nv_bfloat16* x, int64_t ldx, uint8_t* q,
                                                                      float* scale, int K) {
    __shared__ float red[4];
    const int64_t row = blockIdx.x;
    const uint4* xin = reinterpret_cast<const uint4*>(x + row * ldx);
    const int nvec = K >> 3;
    uint4 v[V];
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < V; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) {
            v[j] = xin[i];
            amax = absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(amax, v[j].x), v[j].y), v[j].z), v[j].w);
        }
    }
    const float s = fp8_row_scale(row_block_max(amax, red));
    if (threadIdx.x == 0) scale[row] = s;
    uint2* o = reinterpret_cast<uint2*>(q + row * K);
#pragma unroll
    for (int j = 0; j < V; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) o[i] = quant_bf16x8(v[j], s);
    }
}

struct LnModParams {
    const __nv_bfloat16* x;      // input rows
    __nv_bfloat16* out;          // output rows [B*rows_out, D] (bf16 form)
    uint8_t* out_q;              // fp8 form: e4m3 rows [B*rows_out, D] and their fp32 scales [B*rows_out]
    float* out_scale;
    const __nv_bfloat16* gamma;  // optional affine
    const __nv_bfloat16* beta;
    const __nv_bfloat16* shift;  // optional modulation [B, mod_stride]
    const __nv_bfloat16* scale;
    int64_t mod_stride;
    int D;
    int rows_out;         // rows per batch written
    int in_batch_rows;    // rows per batch in the input
    int in_row_offset;    // first input row (within a batch) to read
    int total_rows;       // B * rows_out
    float eps;
};

// bf16x2 word -> f32x2 pair (two ALU ops: shift and mask instead of two conversions).
__device__ __forceinline__ uint64_t bf16x2_to_f32x2(uint32_t w) {
    return pack_f32x2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
__device__ __forceinline__ uint64_t mul_f32x2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack_f32x2(a, a0, a1);
    unpack_f32x2(b, b0, b1);
    return pack_f32x2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint32_t f32x2_to_bf16x2(uint64_t v) {
    float lo, hi;
    unpack_f32x2(v, lo, hi);
    return pack_bf16(lo, hi);
}
__device__ __forceinline__ float hsum_f32x2(uint64_t v) {
    float lo, hi;
    unpack_f32x2(v, lo, hi);
    return lo + hi;
}

// LayerNorm (+optional affine) (+optional AdaLN modulate x*(1+scale)+shift).
// Restates F.layer_norm + modulate (dit_video_crossattn_sc_xc.py:760-761, :1031-1032, :1045-1046, :825).
// The row is unpacked to fp32 pairs once and stays in registers (4 x ROW_MAXV packed f32x2 per thread) for all three passes.
// FP8: the bf16 row the bf16 form would write is quantised to e4m3 in registers (one more block reduction for its amax),
// so the result equals quant_rows_fp8 of the bf16 form bit for bit.
template <bool FP8>
__global__ void __launch_bounds__(ROW_THREADS) ln_modulate_kernel(const LnModParams p) {
    __shared__ float red[4];
    const int row = blockIdx.x;
    const int b = row / p.rows_out;
    const int r = row - b * p.rows_out;
    const int64_t in_row = static_cast<int64_t>(b) * p.in_batch_rows + p.in_row_offset + r;
    const uint4* xin = reinterpret_cast<const uint4*>(p.x + in_row * p.D);
    const int nvec = p.D >> 3;  // 16-byte vectors in the row
    uint64_t x[ROW_MAXV][4];
    uint64_t acc = 0ull;
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) {
            const uint4 v = xin[i];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                x[j][k] = bf16x2_to_f32x2(w[k]);
                acc = add_f32x2(acc, x[j][k]);
            }
        }
    }
    const float mean = row_block_sum(hsum_f32x2(acc), red) / p.D;
    const uint64_t nmean2 = pack_f32x2(-mean, -mean);
    acc = 0ull;
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        if (j * ROW_THREADS + threadIdx.x < nvec) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                x[j][k] = add_f32x2(x[j][k], nmean2);  // centred
                acc = fma_f32x2(x[j][k], x[j][k], acc);
            }
        }
    }
    const float rstd = rsqrtf(row_block_sum(hsum_f32x2(acc), red) / p.D + p.eps);
    const uint64_t rstd2 = pack_f32x2(rstd, rstd), one2 = pack_f32x2(1.0f, 1.0f);
    uint4* o = reinterpret_cast<uint4*>(p.out + static_cast<int64_t>(row) * p.D);
    [[maybe_unused]] uint4 ob[ROW_MAXV];  // fp8: the bf16 row, kept for the quantisation
    [[maybe_unused]] float amax = 0.f;
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) {
            const int col = i * 8;
            uint64_t y[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) y[k] = mul_f32x2(x[j][k], rstd2);
            if (p.gamma) {
                const uint4 g = *reinterpret_cast<const uint4*>(p.gamma + col);
                const uint4 bb = *reinterpret_cast<const uint4*>(p.beta + col);
                const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, bw[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) y[k] = fma_f32x2(y[k], bf16x2_to_f32x2(gw[k]), bf16x2_to_f32x2(bw[k]));
            }
            if (p.scale) {
                const uint4 sc = *reinterpret_cast<const uint4*>(p.scale + b * p.mod_stride + col);
                const uint4 sh = *reinterpret_cast<const uint4*>(p.shift + b * p.mod_stride + col);
                const uint32_t sw[4] = {sc.x, sc.y, sc.z, sc.w}, hw[4] = {sh.x, sh.y, sh.z, sh.w};
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    y[k] = fma_f32x2(y[k], add_f32x2(one2, bf16x2_to_f32x2(sw[k])), bf16x2_to_f32x2(hw[k]));
            }
            uint4 ov;
            ov.x = f32x2_to_bf16x2(y[0]);
            ov.y = f32x2_to_bf16x2(y[1]);
            ov.z = f32x2_to_bf16x2(y[2]);
            ov.w = f32x2_to_bf16x2(y[3]);
            if constexpr (FP8) {
                ob[j] = ov;
                amax = absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(amax, ov.x), ov.y), ov.z), ov.w);
            } else {
                o[i] = ov;
            }
        }
    }
    if constexpr (FP8) {
        const float s = fp8_row_scale(row_block_max(amax, red));
        if (threadIdx.x == 0) p.out_scale[row] = s;
        uint2* oq = reinterpret_cast<uint2*>(p.out_q + static_cast<int64_t>(row) * p.D);
#pragma unroll
        for (int j = 0; j < ROW_MAXV; ++j) {
            const int i = j * ROW_THREADS + threadIdx.x;
            if (i < nvec) oq[i] = quant_bf16x8(ob[j], s);
        }
    }
}

struct RmsRopeParams {
    __nv_bfloat16* buf;   // [rows, ld] ; normalised in place
    int64_t ld;
    int col_offset[2];    // column offset of slab 0 / slab 1 (e.g. q and k inside the fused QKV buffer)
    const __nv_bfloat16* weight[2];
    int nslabs;           // 1 or 2
    int D;                // normalised width (hidden size), D % 8 == 0 (D % 128 == 0 with RoPE)
    int rows;             // total rows (B * rows_per_batch)
    int rows_per_batch;
    const float* cos;     // optional [rows_per_batch, 128] fp32 tables (token = row % rows_per_batch)
    const float* sin;
    float eps;
};

// RMSNorm over the full hidden width (dit_video_crossattn_sc_xc.py:61-68, F5) fused with the
// interleaved-pair 3-D RoPE (:336-340, :525-645).  grid.y selects the slab (q / k).
__global__ void __launch_bounds__(ROW_THREADS) rmsnorm_rope_kernel(const RmsRopeParams p) {
    __shared__ float red[4];
    const int row = blockIdx.x;
    const int slab = blockIdx.y;
    __nv_bfloat16* base = p.buf + static_cast<int64_t>(row) * p.ld + (slab ? p.col_offset[1] : p.col_offset[0]);
    uint4* xin = reinterpret_cast<uint4*>(base);
    const int nvec = p.D >> 3;
    uint64_t x[ROW_MAXV][4];  // the row as packed fp32 pairs (pair = one interleaved RoPE pair)
    uint64_t acc = 0ull;
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) {
            const uint4 v = xin[i];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                x[j][k] = bf16x2_to_f32x2(w[k]);
                acc = fma_f32x2(x[j][k], x[j][k], acc);
            }
        }
    }
    // head_dim = 128 = 16 vectors and ROW_THREADS % 16 == 0: the rope column (col % 128) of a thread is (tid % 16) * 8
    // for every vector it owns, so one (cos, sin) octet per thread serves the whole row; fetched before the reduction
    // so that its latency hides behind it.  out pair = (x1, x2) * (c0, c1) + (x2, x1) * (-s0, s1)   (:336-340)
    uint64_t c2[4], s2[4];
    const bool rope = p.cos != nullptr;
    if (rope) {
        const int tok = row % p.rows_per_batch;
        const float4* c4 = reinterpret_cast<const float4*>(p.cos + static_cast<int64_t>(tok) * 128 + (threadIdx.x & 15) * 8);
        const float4* s4 = reinterpret_cast<const float4*>(p.sin + static_cast<int64_t>(tok) * 128 + (threadIdx.x & 15) * 8);
        const float4 ca = c4[0], cb = c4[1], sa = s4[0], sb = s4[1];
        c2[0] = pack_f32x2(ca.x, ca.y); c2[1] = pack_f32x2(ca.z, ca.w); c2[2] = pack_f32x2(cb.x, cb.y); c2[3] = pack_f32x2(cb.z, cb.w);
        s2[0] = pack_f32x2(-sa.x, sa.y); s2[1] = pack_f32x2(-sa.z, sa.w); s2[2] = pack_f32x2(-sb.x, sb.y); s2[3] = pack_f32x2(-sb.z, sb.w);
    }
    const float rstd = rsqrtf(row_block_sum(hsum_f32x2(acc), red) / p.D + p.eps);
    const uint64_t rstd2 = pack_f32x2(rstd, rstd);
    const __nv_bfloat16* wgt = slab ? p.weight[1] : p.weight[0];  // (a dynamic index would spill the param arrays to local memory)
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) {
            const uint4 g = *reinterpret_cast<const uint4*>(wgt + i * 8);
            const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
            uint32_t ow[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                uint64_t y = mul_f32x2(bf16x2_to_f32x2(gw[k]), mul_f32x2(x[j][k], rstd2));  // g * (x * rstd), as the reference orders it
                if (rope) {
                    float y1, y2;
                    unpack_f32x2(y, y1, y2);
                    y = fma_f32x2(pack_f32x2(y2, y1), s2[k], mul_f32x2(y, c2[k]));
                }
                ow[k] = f32x2_to_bf16x2(y);
            }
            xin[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
    }
}

// mod[b, i] = emb[b, i] + param[i]   (dit_video_crossattn_sc_xc.py:1025-1028, :823) fp32 add, one bf16 rounding
__global__ void adaln_modulation_kernel(const __nv_bfloat16* emb, const __nv_bfloat16* param, __nv_bfloat16* out,
                                        int B, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * n) return;
    out[i] = __float2bfloat16(__bfloat162float(emb[i]) + __bfloat162float(param[i % n]));
}

__global__ void silu_kernel(const __nv_bfloat16* x, __nv_bfloat16* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = __bfloat162float(x[i]);
    out[i] = __float2bfloat16(v / (1.0f + expf(-v)));
}

// sgm/modules/diffusionmodules/util.py:207-231: freqs in fp64, args fp32, cos||sin, cast to bf16
__global__ void timestep_embedding_kernel(const float* t, __nv_bfloat16* out, int B, int dim) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int half = dim / 2;
    if (i >= B * half) return;
    const int b = i / half, k = i - b * half;
    const double fr = exp(-log(10000.0) * static_cast<double>(k) / static_cast<double>(half));
    const float arg = t[b] * static_cast<float>(fr);
    out[b * dim + k] = __float2bfloat16(cosf(arg));
    out[b * dim + half + k] = __float2bfloat16(sinf(arg));
}

struct PatchifyParams {
    const __nv_bfloat16* x;     // [B, T, cin, H, W]
    const __nv_bfloat16* ref;   // [Br, 1, cin, H, W]
    const __nv_bfloat16* pose;  // [Bp, T, cin, H/2, W/2]
    __nv_bfloat16* a_main;      // [B, (1+T)*H/2*W/2, 80]   rows: ref tokens then noise tokens
    __nv_bfloat16* a_pose;      // [B, T*H/4*W/4, 80]
    int B, Br, Bp, T, H, W;
    int cin;  // channels present in the inputs: 16 (mask channels synthesised) or 20 (already appended)
};

// Patch gather for the two Conv3d(20->d, k=s=(1,2,2)) of ImagePatchEmbeddingMixin
// (dit_video_crossattn_sc_xc.py:99-130) incl. the mask channels appended in
// DiffusionTransformer.forward (:1468, :1483-1486, :1496-1503): x gets 4 zero channels,
// ref and pose get 4 one channels.  A[token, c*4 + p*2 + q] = in[b, t, c, 2y+p, 2x+q].
__global__ void patchify_kernel(const PatchifyParams p) {
    const int hp = p.H / 2, wp = p.W / 2, hq = p.H / 4, wq = p.W / 4;
    const int n_main = (1 + p.T) * hp * wp, n_pose = p.T * hq * wq;
    const int64_t total = static_cast<int64_t>(p.B) * (n_main + n_pose) * 20;
    int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = i % 20;
    int64_t tok = i / 20;
    const int b = tok / (n_main + n_pose);
    int n = tok - static_cast<int64_t>(b) * (n_main + n_pose);
    const __nv_bfloat16 one = __float2bfloat16(1.0f), zero = __float2bfloat16(0.0f);
    __nv_bfloat16 v[4];
    __nv_bfloat16* dst;
    if (n < n_main) {
        const int t = n / (hp * wp), rem = n - t * hp * wp, y = rem / wp, x = rem - y * wp;
        dst = p.a_main + (static_cast<int64_t>(b) * n_main + n) * 80 + c * 4;
        if (c >= p.cin) {
            const __nv_bfloat16 m = (t == 0) ? one : zero;
            v[0] = v[1] = v[2] = v[3] = m;
        } else {
            const __nv_bfloat16* src =
                (t == 0) ? p.ref + ((static_cast<int64_t>(b % p.Br) * p.cin + c) * p.H) * p.W
                         : p.x + (((static_cast<int64_t>(b) * p.T + (t - 1)) * p.cin + c) * p.H) * p.W;
            v[0] = src[(2 * y) * p.W + 2 * x];
            v[1] = src[(2 * y) * p.W + 2 * x + 1];
            v[2] = src[(2 * y + 1) * p.W + 2 * x];
            v[3] = src[(2 * y + 1) * p.W + 2 * x + 1];
        }
    } else {
        n -= n_main;
        const int t = n / (hq * wq), rem = n - t * hq * wq, y = rem / wq, x = rem - y * wq;
        dst = p.a_pose + (static_cast<int64_t>(b) * n_pose + n) * 80 + c * 4;
        if (c >= p.cin) {
            v[0] = v[1] = v[2] = v[3] = one;
        } else {
            const int H2 = p.H / 2, W2 = p.W / 2;
            const __nv_bfloat16* src = p.pose + (((static_cast<int64_t>(b % p.Bp) * p.T + t) * p.cin + c) * H2) * W2;
            v[0] = src[(2 * y) * W2 + 2 * x];
            v[1] = src[(2 * y) * W2 + 2 * x + 1];
            v[2] = src[(2 * y + 1) * W2 + 2 * x];
            v[3] = src[(2 * y + 1) * W2 + 2 * x + 1];
        }
    }
    uint2 o;
    o.x = static_cast<uint32_t>(__bfloat16_as_ushort(v[0])) | (static_cast<uint32_t>(__bfloat16_as_ushort(v[1])) << 16);
    o.y = static_cast<uint32_t>(__bfloat16_as_ushort(v[2])) | (static_cast<uint32_t>(__bfloat16_as_ushort(v[3])) << 16);
    *reinterpret_cast<uint2*>(dst) = o;
}

// unpatchify (dit_video_crossattn_sc_xc.py:764-784): lin [B, T*Hp*Wp, 64] with feature order (p q c)
//   -> out [B, T, 16, 2*Hp, 2*Wp]
__global__ void unpatchify_kernel(const __nv_bfloat16* lin, __nv_bfloat16* out, int B, int T, int Hp, int Wp) {
    const int64_t total = static_cast<int64_t>(B) * T * 16 * (2 * Hp) * (2 * Wp);
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int W = 2 * Wp, H = 2 * Hp;
    const int xx = i % W;
    const int yy = (i / W) % H;
    const int c = (i / (static_cast<int64_t>(W) * H)) % 16;
    const int t = (i / (static_cast<int64_t>(W) * H * 16)) % T;
    const int b = i / (static_cast<int64_t>(W) * H * 16 * T);
    const int y = yy >> 1, pp = yy & 1, x = xx >> 1, q = xx & 1;
    const int64_t tok = (static_cast<int64_t>(b) * T + t) * Hp * Wp + y * Wp + x;
    out[i] = lin[tok * 64 + (pp * 2 + q) * 16 + c];
}

// VanillaCFG + Euler update, fp32 (guiders.py:41-45, sampling_utils.py:7-10, sampling.py:960-963):
// x += dsigma * (u + s*(c-u)), model output v is bf16 [2, n] (uncond, cond)
__global__ void cfg_euler_kernel(float* x, const __nv_bfloat16* v, int64_t n, float scale, float dsigma) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float u = __bfloat162float(v[i]), c = __bfloat162float(v[n + i]);
    x[i] = x[i] + dsigma * (u + scale * (c - u));
}

__global__ void cast_f32_to_bf16_kernel(const float* x, __nv_bfloat16* out, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __float2bfloat16(x[i]);
}

}  // namespace scail
