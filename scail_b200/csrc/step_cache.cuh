// First-block residual cache (scail_b200/step_cache.py): the three HBM-bound passes around the skipped blocks.
// All tensors are bf16 [B, N, d] token rows (ref || noise || pose per batch element) except R, fp32 [B, n_seq, d] over the
// noise rows only.  Every thread moves whole 16-byte vectors (8 bf16), so d % 8 == 0 and the pointers are 16-byte aligned.
#pragma once
#include <cuda_bf16.h>

#include "rowops.cuh"  // warp_sum

namespace scail {

constexpr int SC_THREADS = 256;
constexpr int SC_MAX_CTAS = 1024;  // the indicator's fixed grid cap: partials hold 2 * SC_MAX_CTAS floats

__device__ __forceinline__ void sc_unpack(const uint4& u, float (&f)[8]) {
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __bfloat1622float2(p[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

__device__ __forceinline__ uint4 sc_pack(const float (&f)[8]) {
    uint4 u;
    __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    return u;
}

// Vector v of a [B, n_seq, d] noise-row tensor -> its vector in the [B, N, d] tensor (row offset n_ref per batch element).
// The host guarantees B * N * d / 8 < 2^31, so 32-bit division is exact.
__device__ __forceinline__ int64_t sc_noise_to_full(unsigned v, unsigned vpr, unsigned n_seq, unsigned N, unsigned n_ref) {
    const unsigned row = v / vpr, c = v - row * vpr;
    const unsigned b = row / n_seq, n = row - b * n_seq;
    return (static_cast<int64_t>(b) * N + n_ref + n) * vpr + c;
}

// Pass 1's CTA epilogue: this thread's fp32 sums a and b, summed over the CTA in a fixed order (warp shuffle tree, then
// the warps in index order) -> partials[blockIdx.x] and partials[gridDim.x + blockIdx.x].  Every thread of the CTA calls it.
__device__ __forceinline__ void sc_write_partials(float s_a, float s_b, float* __restrict__ partials) {
    __shared__ float red[2][SC_THREADS / 32];
    s_a = warp_sum(s_a);
    s_b = warp_sum(s_b);
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = s_a;
        red[1][threadIdx.x >> 5] = s_b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int w = 0; w < SC_THREADS / 32; ++w) {
            a += red[0][w];
            b += red[1][w];
        }
        partials[blockIdx.x] = a;
        partials[gridDim.x + blockIdx.x] = b;
    }
}

// Pass 1 of the indicator.  r = bf16_rn(f32(h1) - f32(h0)) -> r_new; h1's noise rows -> h1c; this CTA's fp32 partial sums
// of |r - r_ref| and |r_ref| -> partials[blockIdx.x] and partials[gridDim.x + blockIdx.x].  The grid is a function of the
// shape only and every thread walks the same grid-stride vectors in the same order, so the partials do not depend on the
// device, the stream or timing.
__global__ void __launch_bounds__(SC_THREADS) step_cache_indicator_kernel(
    const uint4* __restrict__ h0, const uint4* __restrict__ h1, const uint4* __restrict__ r_ref, uint4* __restrict__ r_new,
    uint4* __restrict__ h1c, float* __restrict__ partials, int64_t nvec, unsigned vpr, unsigned N, int n_ref, int n_seq) {
    float s_diff = 0.f, s_ref = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * SC_THREADS;
    for (int64_t v = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x; v < nvec; v += stride) {
        const uint4 a = h0[v], b = h1[v], c = r_ref[v];
        float fa[8], fb[8], fc[8], fr[8];
        sc_unpack(a, fa);
        sc_unpack(b, fb);
        sc_unpack(c, fc);
#pragma unroll
        for (int i = 0; i < 8; ++i) fr[i] = fb[i] - fa[i];
        const uint4 r = sc_pack(fr);
        r_new[v] = r;
        sc_unpack(r, fr);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            s_diff += fabsf(fr[i] - fc[i]);
            s_ref += fabsf(fc[i]);
        }
        const unsigned row = static_cast<unsigned>(v) / vpr, bb = row / N;
        const int n = static_cast<int>(row - bb * N) - n_ref;
        if (n >= 0 && n < n_seq)
            h1c[(static_cast<int64_t>(bb) * n_seq + n) * vpr + (static_cast<unsigned>(v) - row * vpr)] = b;
    }
    sc_write_partials(s_diff, s_ref, partials);
}

// The two fp64 sums of n_parts partial pairs (partials[i] and partials[n_parts + i]) by one CTA of SC_THREADS threads, in a
// fixed order; thread 0 gets them in red[0][0] and red[1][0].  Shared by every pass 2 of a two-pass reduction.
__device__ __forceinline__ void sc_sum_partials(const float* __restrict__ partials, int n_parts, double (&red)[2][SC_THREADS]) {
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < n_parts; i += SC_THREADS) {
        a += static_cast<double>(partials[i]);
        b += static_cast<double>(partials[n_parts + i]);
    }
    red[0][threadIdx.x] = a;
    red[1][threadIdx.x] = b;
    __syncthreads();
    for (int s = SC_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            red[0][threadIdx.x] += red[0][threadIdx.x + s];
            red[1][threadIdx.x] += red[1][threadIdx.x + s];
        }
        __syncthreads();
    }
}

// Pass 2: one CTA sums the n_parts partials in fp64 in a fixed order -> out = {sum|r - r_ref|, sum|r_ref|, ratio, 0}; the
// ratio is +inf when the denominator is zero (and NaN propagates).
__global__ void __launch_bounds__(SC_THREADS) step_cache_finish_kernel(const float* __restrict__ partials, int n_parts,
                                                                       double* __restrict__ out) {
    __shared__ double red[2][SC_THREADS];
    sc_sum_partials(partials, n_parts, red);
    if (threadIdx.x == 0) {
        const double num = red[0][0], den = red[1][0];
        out[0] = num;
        out[1] = den;
        out[2] = den == 0.0 ? static_cast<double>(INFINITY) : num / den;
        out[3] = 0.0;
    }
}

// R = f32(h[noise rows]) - f32(h1c), one 8-element vector per thread.
__global__ void __launch_bounds__(SC_THREADS) step_cache_update_kernel(const uint4* __restrict__ h, const uint4* __restrict__ h1c,
                                                                       float4* __restrict__ R, int64_t nvec, int vpr, int N,
                                                                       int n_ref, int n_seq) {
    const int64_t v = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x;
    if (v >= nvec) return;
    float fh[8], fc[8];
    sc_unpack(h[sc_noise_to_full(v, vpr, n_seq, N, n_ref)], fh);
    sc_unpack(h1c[v], fc);
    R[2 * v] = make_float4(fh[0] - fc[0], fh[1] - fc[1], fh[2] - fc[2], fh[3] - fc[3]);
    R[2 * v + 1] = make_float4(fh[4] - fc[4], fh[5] - fc[5], fh[6] - fc[6], fh[7] - fc[7]);
}

// In place on the noise rows: h = bf16_rn(f32(h) + R), one 8-element vector per thread.
__global__ void __launch_bounds__(SC_THREADS) step_cache_apply_kernel(uint4* __restrict__ h, const float4* __restrict__ R,
                                                                      int64_t nvec, int vpr, int N, int n_ref, int n_seq) {
    const int64_t v = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x;
    if (v >= nvec) return;
    const int64_t dst = sc_noise_to_full(v, vpr, n_seq, N, n_ref);
    float f[8];
    sc_unpack(h[dst], f);
    const float4 r0 = R[2 * v], r1 = R[2 * v + 1];
    f[0] += r0.x; f[1] += r0.y; f[2] += r0.z; f[3] += r0.w;
    f[4] += r1.x; f[5] += r1.y; f[6] += r1.z; f[7] += r1.w;
    h[dst] = sc_pack(f);
}

// ---- Taylor forecast (FirstBlockCache(order >= 1)): n_slots fp32 residual slots [B, n_seq, d], slot s at R + s * slot_stride.
// The slot index and the coefficients are read from device memory, so one captured graph serves every step.
constexpr int SC_MAX_SLOTS = 3;

// R[*slot] = f32(h[noise rows]) - f32(h1c) (step_cache_update's arithmetic); a slot outside [0, n_slots) writes nothing.
__global__ void __launch_bounds__(SC_THREADS) step_cache_update_slot_kernel(const uint4* __restrict__ h,
                                                                            const uint4* __restrict__ h1c, float* __restrict__ R,
                                                                            int64_t slot_stride, int n_slots,
                                                                            const int* __restrict__ slot, int64_t nvec, int vpr,
                                                                            int N, int n_ref, int n_seq) {
    const int s = *slot;
    const int64_t v = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x;
    if (s < 0 || s >= n_slots || v >= nvec) return;
    float4* Rs = reinterpret_cast<float4*>(R + s * slot_stride);
    float fh[8], fc[8];
    sc_unpack(h[sc_noise_to_full(v, vpr, n_seq, N, n_ref)], fh);
    sc_unpack(h1c[v], fc);
    Rs[2 * v] = make_float4(fh[0] - fc[0], fh[1] - fc[1], fh[2] - fc[2], fh[3] - fc[3]);
    Rs[2 * v + 1] = make_float4(fh[4] - fc[4], fh[5] - fc[5], fh[6] - fc[6], fh[7] - fc[7]);
}

// In place on the noise rows: t = c0*R0, t = t + c1*R1, t = t + c2*R2 (slot order, every product and sum rounded on its
// own: no FMA contraction), then h = bf16_rn(f32(h) + t).  A slot whose coefficient is exactly 0 is neither read nor
// added, so stale or NaN slots cannot leak in and c = (1, 0, 0) is step_cache_apply bit for bit; with no active slot h
// is left as it is.
__global__ void __launch_bounds__(SC_THREADS) step_cache_apply_forecast_kernel(uint4* __restrict__ h, const float* __restrict__ R,
                                                                               int64_t slot_stride, int n_slots,
                                                                               const float* __restrict__ coef, int64_t nvec,
                                                                               int vpr, int N, int n_ref, int n_seq) {
    const int64_t v = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x;
    if (v >= nvec) return;
    float c[SC_MAX_SLOTS];
    bool any = false;
#pragma unroll
    for (int s = 0; s < SC_MAX_SLOTS; ++s) {
        c[s] = s < n_slots ? coef[s] : 0.f;
        any = any || c[s] != 0.f;
    }
    if (!any) return;
    float t[8];
    bool first = true;
#pragma unroll
    for (int s = 0; s < SC_MAX_SLOTS; ++s) {
        if (c[s] == 0.f) continue;
        const float4* Rs = reinterpret_cast<const float4*>(R + s * slot_stride);
        const float4 r0 = Rs[2 * v], r1 = Rs[2 * v + 1];
        const float r[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float p = __fmul_rn(c[s], r[i]);
            t[i] = first ? p : __fadd_rn(t[i], p);
        }
        first = false;
    }
    const int64_t dst = sc_noise_to_full(v, vpr, n_seq, N, n_ref);
    float f[8];
    sc_unpack(h[dst], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = __fadd_rn(f[i], t[i]);
    h[dst] = sc_pack(f);
}

}  // namespace scail
