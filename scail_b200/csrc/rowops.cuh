// HBM-bound row / elementwise kernels of the SCAIL DiT step (everything that is not a GEMM or attention).
// One warp per row, 16-byte vectorised loads, fp32 statistics, bf16 in/out.
#pragma once
#include <cuda_fp8.h>

#include "attention.cuh"  // ATT_D and fp8_vt_key (the V^T pre-pass)
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

// ---- INT8 row format of fp8_attention="int8_qk" (Q and smoothed K) and of fp8_linear="int8" (both GEMM operands):
// s = amax(|row|) / 127 (IEEE division),
// q = cvt.rni.sat.s8(x / s) in [-127, 127]; an all-zero row gets s = 1 and q = 0.
// torch: torch.round(x.float() / s[:, None]).clamp(-127, 127).to(torch.int8)  (round-half-even, as cvt.rni)
constexpr float INT8_QMAX = 127.0f;

__device__ __forceinline__ float int8_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, INT8_QMAX) : 1.0f; }
// 8 fp32 -> 8 int8 codes
__device__ __forceinline__ uint2 quant_f32x8_s8(const float (&f)[8], float s) {
    uint32_t w[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = max(-127, min(127, __float2int_rn(__fdiv_rn(f[i], s))));
        w[i >> 2] |= (static_cast<uint32_t>(q) & 0xffu) << (8 * (i & 3));
    }
    return make_uint2(w[0], w[1]);
}
// 8 bf16 -> 8 int8 codes
__device__ __forceinline__ uint2 quant_bf16x8_s8(const uint4 v, float s) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 x = unpack_bf16(w[k]);
        f[2 * k] = x.x;
        f[2 * k + 1] = x.y;
    }
    return quant_f32x8_s8(f, s);
}

// One 128-thread block per row of a row-strided bf16 [M, K] (K % 16 == 0, K <= 8 * ROW_THREADS * V): the row stays in registers
// between the amax reduction and the quantisation, so it is read once.  INT8: the INT8 row format instead of e4m3.
template <int V, bool INT8>
__device__ __forceinline__ void quant_rows_body(const __nv_bfloat16* x, int64_t ldx, uint8_t* q, float* scale, int K) {
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
    const float s = INT8 ? int8_row_scale(row_block_max(amax, red)) : fp8_row_scale(row_block_max(amax, red));
    if (threadIdx.x == 0) scale[row] = s;
    uint2* o = reinterpret_cast<uint2*>(q + row * K);
#pragma unroll
    for (int j = 0; j < V; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        if (i < nvec) o[i] = INT8 ? quant_bf16x8_s8(v[j], s) : quant_bf16x8(v[j], s);
    }
}

template <int V>
__global__ void __launch_bounds__(ROW_THREADS) quant_rows_fp8_kernel(const __nv_bfloat16* x, int64_t ldx, uint8_t* q,
                                                                      float* scale, int K) {
    quant_rows_body<V, false>(x, ldx, q, scale, K);
}

template <int V>
__global__ void __launch_bounds__(ROW_THREADS) quant_rows_int8_kernel(const __nv_bfloat16* x, int64_t ldx, uint8_t* q,
                                                                       float* scale, int K) {
    quant_rows_body<V, true>(x, ldx, q, scale, K);
}

struct LnModParams {
    const __nv_bfloat16* x;      // input rows
    __nv_bfloat16* out;          // output rows [B*rows_out, D] (bf16 form)
    uint8_t* out_q;              // fp8 / int8 form: e4m3 or int8 rows [B*rows_out, D] and their fp32 scales [B*rows_out]
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
// so the result equals quant_rows_fp8 of the bf16 form bit for bit.  INT8 (FP8 false): the same in the INT8 row format,
// equal to quant_rows_int8 of the bf16 form.
template <bool FP8, bool INT8 = false>
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
    constexpr bool QUANT = FP8 || INT8;
    [[maybe_unused]] uint4 ob[ROW_MAXV];  // fp8 / int8: the bf16 row, kept for the quantisation
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
            if constexpr (QUANT) {
                ob[j] = ov;
                amax = absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(amax, ov.x), ov.y), ov.z), ov.w);
            } else {
                o[i] = ov;
            }
        }
    }
    if constexpr (QUANT) {
        const float s = INT8 ? int8_row_scale(row_block_max(amax, red)) : fp8_row_scale(row_block_max(amax, red));
        if (threadIdx.x == 0) p.out_scale[row] = s;
        uint2* oq = reinterpret_cast<uint2*>(p.out_q + static_cast<int64_t>(row) * p.D);
#pragma unroll
        for (int j = 0; j < ROW_MAXV; ++j) {
            const int i = j * ROW_THREADS + threadIdx.x;
            if (i < nvec) oq[i] = INT8 ? quant_bf16x8_s8(ob[j], s) : quant_bf16x8(ob[j], s);
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
    // fp8 form (rmsnorm_rope_kernel<true>): slab s goes to e4m3 rows q8[s] [rows, ld8] (buf is not written) with one fp32
    // scale per (token, head) in s8[s], head-major [B, H, L_pad] (rows_per_batch = L tokens; [L, L_pad) written as zeros)
    uint8_t* q8[2];
    float* s8[2];
    int64_t ld8;
    int L_pad;
};

// RMSNorm over the full hidden width (dit_video_crossattn_sc_xc.py:61-68, F5) fused with the
// interleaved-pair 3-D RoPE (:336-340, :525-645).  grid.y selects the slab (q / k).
// FP8: the bf16 row the bf16 form would write is quantised per 128-wide head (the e4m3 row format above, one row = one head of
// one token), so the result equals quant_rows_fp8 of the bf16 form's heads bit for bit.  A head's 16 vectors are held by 16
// consecutive lanes (D % 128 == 0), so its amax is four shuffles.
// INT8Q (FP8 false): slab 0 (Q) is quantised the same way in the INT8 row format; slab 1 (K) is written back in bf16 in place,
// exactly as the bf16 form writes it, because its smoothing (quant_k_int8) needs the mean over all keys first.
template <bool FP8, bool INT8Q = false>
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
    [[maybe_unused]] uint4 ob[ROW_MAXV];  // fp8: the bf16 row, kept for the quantisation
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
            if constexpr (FP8) ob[j] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            else if constexpr (INT8Q) {
                if (slab == 0) ob[j] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                else xin[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            } else xin[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
    }
    if constexpr (FP8 || INT8Q) {
        if (INT8Q && slab == 1) return;  // the whole block: K went back in bf16
        uint8_t* q8 = (slab ? p.q8[1] : p.q8[0]) + static_cast<int64_t>(row) * p.ld8;
        float* s8 = slab ? p.s8[1] : p.s8[0];
        const int b = row / p.rows_per_batch, tok = row - b * p.rows_per_batch;
        const int heads = p.D >> 7;
#pragma unroll
        for (int j = 0; j < ROW_MAXV; ++j) {
            const int i = j * ROW_THREADS + threadIdx.x;
            // all lanes shuffle (a lane past the row contributes 0); the 16 lanes of a head are all in or all out
            float amax = 0.f;
            if (i < nvec) amax = absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(absmax_bf16x2(0.f, ob[j].x), ob[j].y), ob[j].z), ob[j].w);
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            if (i < nvec) {
                const float s = INT8Q ? int8_row_scale(amax) : fp8_row_scale(amax);
                reinterpret_cast<uint2*>(q8)[i] = INT8Q ? quant_bf16x8_s8(ob[j], s) : quant_bf16x8(ob[j], s);
                if ((i & 15) == 0) {
                    float* sh = s8 + (static_cast<int64_t>(b) * heads + (i >> 4)) * p.L_pad;
                    sh[tok] = s;
                    for (int pad = p.rows_per_batch + tok; pad < p.L_pad; pad += p.rows_per_batch) sh[pad] = 0.f;
                }
            }
        }
    }
}

// ---- K of fp8_attention="int8_qk": smoothing + INT8 quantisation (scail_quant_k_int8), three launches, no atomics:
//   k_mean_partial_kernel : per (batch, 256-key chunk, channel) the fp64 sum of the chunk's bf16 keys, in ascending key order;
//   k_mean_finish_kernel  : k-bar[b, c] = f32((sum of the chunks' partials in ascending chunk order) / L), fp64 throughout;
//   quant_k_int8_kernel   : K'[row] = __fsub_rn(f32(k), k-bar) in registers, quantised per 128-wide head in the INT8 row
//                           format: codes [B*L, ld8], scales head-major [B, H, L_pad] with zeros past L.
// The partition is fixed by the shape, so every launch writes the same bits.
constexpr int KMEAN_ROWS = 256;  // keys per chunk of the partial sums

// grid (ceil(L / 256), B, ceil(D / 1024)), 128 threads: 8 channels per thread
__global__ void __launch_bounds__(128) k_mean_partial_kernel(const __nv_bfloat16* k, int64_t ldk, double* partial, int L, int D) {
    const int b = blockIdx.y;
    const int col = (blockIdx.z * 128 + threadIdx.x) * 8;
    if (col >= D) return;
    const int r0 = blockIdx.x * KMEAN_ROWS, r1 = min(L, r0 + KMEAN_ROWS);
    double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const __nv_bfloat16* src = k + (static_cast<int64_t>(b) * L) * ldk + col;
#pragma unroll 8
    for (int r = r0; r < r1; ++r) {
        const uint4 x = *reinterpret_cast<const uint4*>(src + static_cast<int64_t>(r) * ldk);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = unpack_bf16(w[i]);
            acc[2 * i] += static_cast<double>(f.x);
            acc[2 * i + 1] += static_cast<double>(f.y);
        }
    }
    double* dst = partial + (static_cast<int64_t>(b) * gridDim.x + blockIdx.x) * D + col;
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = acc[i];
}

// grid (ceil(D / 128), B), one thread per channel
__global__ void __launch_bounds__(128) k_mean_finish_kernel(const double* partial, float* kbar, int n_chunks, int L, int D) {
    const int b = blockIdx.y, c = blockIdx.x * 128 + threadIdx.x;
    if (c >= D) return;
    const double* src = partial + static_cast<int64_t>(b) * n_chunks * D + c;
    double acc = 0.0;
    for (int i = 0; i < n_chunks; ++i) acc += src[static_cast<int64_t>(i) * D];
    kbar[static_cast<int64_t>(b) * D + c] = static_cast<float>(acc / static_cast<double>(L));
}

// One 128-thread block per key row (rows = B * L), D = H * 128 <= ROW_MAXV * 1024
__global__ void __launch_bounds__(ROW_THREADS) quant_k_int8_kernel(const __nv_bfloat16* k, int64_t ldk, const float* kbar,
                                                                    int8_t* k8, int64_t ld8, float* scale, int L, int L_pad,
                                                                    int D) {
    const int row = blockIdx.x;
    const int b = row / L, tok = row - b * L;
    const int heads = D >> 7, nvec = D >> 3;
    const uint4* xin = reinterpret_cast<const uint4*>(k + static_cast<int64_t>(row) * ldk);
    const float* kb = kbar + static_cast<int64_t>(b) * D;
#pragma unroll
    for (int j = 0; j < ROW_MAXV; ++j) {
        const int i = j * ROW_THREADS + threadIdx.x;
        float f[8];
        float amax = 0.f;  // all lanes shuffle (a lane past the row contributes 0); a head's 16 lanes are all in or all out
        if (i < nvec) {
            const uint4 v = xin[i];
            const float4 m0 = reinterpret_cast<const float4*>(kb)[2 * i], m1 = reinterpret_cast<const float4*>(kb)[2 * i + 1];
            const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float2 x = unpack_bf16(w[c]);
                f[2 * c] = __fsub_rn(x.x, m[2 * c]);
                f[2 * c + 1] = __fsub_rn(x.y, m[2 * c + 1]);
            }
#pragma unroll
            for (int c = 0; c < 8; ++c) amax = fmaxf(amax, fabsf(f[c]));
        }
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (i < nvec) {
            const float s = int8_row_scale(amax);
            reinterpret_cast<uint2*>(k8 + static_cast<int64_t>(row) * ld8)[i] = quant_f32x8_s8(f, s);
            if ((i & 15) == 0) {
                float* sh = scale + (static_cast<int64_t>(b) * heads + (i >> 4)) * L_pad;
                sh[tok] = s;
                for (int pad = L + tok; pad < L_pad; pad += L) sh[pad] = 0.f;
            }
        }
    }
}

// ---- V^T pre-pass of the fp8 self-attention (attention_fp8_kernel): V [B*L, H*128] bf16 (a column slab, row pitch ldv) ->
// V^T e4m3 [B, H, 128, L_pad] with one scale per (batch, channel) over the L keys, keys permuted by fp8_vt_key inside every
// 16-key group, zeros at keys >= L.  Two launches after a memset of `amax` ([B, H*128] fp32 bits):
//   quant_vt_amax_kernel : per-channel amax by atomicMax on the bits of non-negative floats (order-independent: deterministic);
//   quant_vt_fp8_kernel  : scale = amax / 448 (1 for an all-zero channel), tiled transpose + quantisation.
constexpr int VT_AMAX_ROWS = 256;  // tokens per block of the amax pass

__global__ void __launch_bounds__(128) quant_vt_amax_kernel(const __nv_bfloat16* v, int64_t ldv, unsigned* amax, int L, int D) {
    const int b = blockIdx.y;
    const int col = (blockIdx.z * 128 + threadIdx.x) * 8;
    if (col >= D) return;
    const int r0 = blockIdx.x * VT_AMAX_ROWS, r1 = min(L, r0 + VT_AMAX_ROWS);
    float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const __nv_bfloat16* src = v + (static_cast<int64_t>(b) * L) * ldv + col;
    for (int r = r0; r < r1; ++r) {
        const uint4 x = *reinterpret_cast<const uint4*>(src + static_cast<int64_t>(r) * ldv);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = unpack_bf16(w[k]);
            m[2 * k] = fmaxf(m[2 * k], fabsf(f.x));
            m[2 * k + 1] = fmaxf(m[2 * k + 1], fabsf(f.y));
        }
    }
    unsigned* dst = amax + static_cast<int64_t>(b) * D + col;
#pragma unroll
    for (int k = 0; k < 8; ++k) atomicMax(dst + k, __float_as_uint(m[k]));
}

constexpr int VT_KEYS = 64;  // keys per block of the transpose pass

// grid (L_pad / 64, H, B), 256 threads: 64 keys x 128 channels of one head through shared memory
__global__ void __launch_bounds__(256) quant_vt_fp8_kernel(const __nv_bfloat16* v, int64_t ldv, const unsigned* amax,
                                                            uint8_t* vt, float* v_scale, int L, int L_pad, int H) {
    __shared__ __nv_bfloat16 tile[VT_KEYS][ATT_D + 8];
    __shared__ float sc[ATT_D];
    const int h = blockIdx.y, b = blockIdx.z;
    const int k0 = blockIdx.x * VT_KEYS;
    const int64_t bh = static_cast<int64_t>(b) * H + h;
    if (threadIdx.x < ATT_D) {
        const float s = fp8_row_scale(__uint_as_float(amax[static_cast<int64_t>(b) * H * ATT_D + h * ATT_D + threadIdx.x]));
        sc[threadIdx.x] = s;
        if (blockIdx.x == 0) v_scale[bh * ATT_D + threadIdx.x] = s;
    }
    // load: 64 keys x 16 vectors of 8 channels, 4 per thread
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int idx = it * 256 + threadIdx.x;
        const int key = idx >> 4, vec = idx & 15;
        uint4 x = make_uint4(0u, 0u, 0u, 0u);
        if (k0 + key < L) x = *reinterpret_cast<const uint4*>(v + (static_cast<int64_t>(b) * L + k0 + key) * ldv + h * ATT_D + vec * 8);
        *reinterpret_cast<uint4*>(&tile[key][vec * 8]) = x;
    }
    __syncthreads();
    // store: channel c = thread / 2, logical keys [32 (thread % 2), +32) of the tile as two 16-byte vectors
    const int c = threadIdx.x >> 1, half = threadIdx.x & 1;
    const float s = sc[c];
    uint4 out[2];
    uint32_t* ow = reinterpret_cast<uint32_t*>(out);
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        float f[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int k = 32 * half + 4 * w + i;
            f[i] = __fdiv_rn(__bfloat162float(tile[fp8_vt_key(k)][c]), s);
        }
        const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(f[0], f[1]), __NV_SATFINITE, __NV_E4M3);
        const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(f[2], f[3]), __NV_SATFINITE, __NV_E4M3);
        ow[w] = lo | (hi << 16);
    }
    uint4* dst = reinterpret_cast<uint4*>(vt + (bh * ATT_D + c) * L_pad + k0 + 32 * half);
    dst[0] = out[0];
    dst[1] = out[1];
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
