// Content-adaptive block-sparse self-attention (scail_b200/sparse.py, AdaptiveTiles): the per-(batch, head) tile maps are
// chosen on the device, per forward, from tile-pooled Q and K, so the whole selection can be captured in a CUDA graph.
//   tile_pool_kernel      : Qbar or Kbar [B, H, n_t, 128] fp32 = the mean of each 128-row tile's valid rows (bf16 slab, or
//                           e4m3 or INT8 slab times its [B, H, L_pad] per-token scales).
//   select_tiles_kernel   : per (b, h, query tile q): s_k = Qbar_q . Kbar_k / sqrt(128), e_k = n_k exp(s_k - max s), keep the
//                           forced tiles (k == q and the tiles holding reference tokens) plus the largest e_k (ties: lower k)
//                           until the kept mass reaches `mass` of the total or `max_tiles` were taken; the row goes to a
//                           bitmask and its count to `counts`.
//   compact_tiles_kernel  : per (b, h) CSR from the bitmasks: kv_tile_ptr[q + 1] = sum of counts[0..q], rows ascending.
// Sums run in a fixed order in fp64 and no atomics are used, so every launch produces the same bits.
#pragma once
#include <cuda_fp8.h>

#include "attention.cuh"  // ATT_D, ATT_BKV

namespace scail {

constexpr int ADA_POOL_UNROLL = 16;      // row loads in flight per thread
constexpr int ADA_SELECT_THREADS = 256;  // 8 warps
constexpr int ADA_MAX_TILES = 2048;      // select_tiles_kernel keeps 20 bytes per key tile in shared memory: L <= 262144

// One CTA per (tile, head, batch), one thread per channel.  x: [B*L, ld] (head h at columns h*128); scale: null for bf16,
// else the e4m3 (kInt8: INT8) operand's per-token scales [B, H, L_pad].  Rows are summed in ascending order in fp64 (exact
// products for e4m3 or int8 x fp32) and the mean rounded once to fp32.  fp8_attention="int8_qk" pools the smoothed K', whose
// s_k of one query tile all shift by the same -Qbar . k-bar: e_k = n_k exp(s_k - max s) and hence the selection do not change.
template <bool kFp8, bool kInt8 = false>
__global__ void __launch_bounds__(ATT_D) tile_pool_kernel(const void* __restrict__ x, int64_t ld, const float* __restrict__ scale,
                                                          float* __restrict__ out, int L, int L_pad, int heads) {
    const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, c = threadIdx.x;
    const int r0 = t * ATT_BKV;
    const int n = min(ATT_BKV, L - r0);
    const int64_t bh = static_cast<int64_t>(b) * heads + h;
    const int64_t base = (static_cast<int64_t>(b) * L + r0) * ld + h * ATT_D + c;
    double acc = 0.0;
    for (int i0 = 0; i0 < n; i0 += ADA_POOL_UNROLL) {
        double v[ADA_POOL_UNROLL];
#pragma unroll
        for (int i = 0; i < ADA_POOL_UNROLL; ++i) {
            v[i] = 0.0;
            if (i0 + i < n) {
                const int64_t off = base + static_cast<int64_t>(i0 + i) * ld;
                if (kInt8) {
                    const int8_t q = static_cast<const int8_t*>(x)[off];
                    v[i] = static_cast<double>(q) * static_cast<double>(scale[bh * L_pad + r0 + i0 + i]);
                } else if (kFp8) {
                    __nv_fp8_e4m3 q;
                    q.__x = static_cast<const __nv_fp8_storage_t*>(x)[off];
                    v[i] = static_cast<double>(static_cast<float>(q)) * static_cast<double>(scale[bh * L_pad + r0 + i0 + i]);
                } else {
                    v[i] = static_cast<double>(__bfloat162float(static_cast<const __nv_bfloat16*>(x)[off]));
                }
            }
        }
#pragma unroll
        for (int i = 0; i < ADA_POOL_UNROLL; ++i) acc += v[i];
    }
    out[(bh * gridDim.x + t) * ATT_D + c] = static_cast<float>(acc / n);
}

struct SelectParams {
    const float* qbar;  // [B, H, n_t, 128]
    const float* kbar;
    int heads, L, n_t, n_ref_tiles;  // n_ref_tiles = ceil(n_ref / 128): the key tiles holding a reference token
    double mass;                     // >= 1: every tile (up to max_tiles taken by mass)
    int max_tiles;                   // tiles taken by mass, at most (-1: no cap)
    int words;                       // ceil(n_t / 32)
    int* counts;                     // scratch [B*H*n_t]: listed tiles per row
    uint32_t* bits;                  // scratch [B*H*n_t, words]: the row as a bitmask
};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One CTA per (query tile, head, batch).  Dynamic shared memory: e [n_t] fp64, sorted [n_t] fp64, rank [n_t] int32.
__global__ void __launch_bounds__(ADA_SELECT_THREADS) select_tiles_kernel(const SelectParams p) {
    extern __shared__ double ada_smem[];
    const int n_t = p.n_t;
    double* e = ada_smem;
    double* sorted = e + n_t;
    int* rank = reinterpret_cast<int*>(sorted + n_t);
    __shared__ double red[ADA_SELECT_THREADS / 32];
    __shared__ int taken;
    const int q = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t bh = static_cast<int64_t>(blockIdx.z) * p.heads + blockIdx.y;
    auto forced = [&](int k) { return k == q || k < p.n_ref_tiles; };

    // s_k = Qbar_q . Kbar_k / sqrt(128): one warp per key tile, four channels per lane
    const float4 qv = reinterpret_cast<const float4*>(p.qbar + (bh * n_t + q) * ATT_D)[lane];
    double smax = -INFINITY;
    for (int k = warp; k < n_t; k += ADA_SELECT_THREADS / 32) {
        const float4 kv = reinterpret_cast<const float4*>(p.kbar + (bh * n_t + k) * ATT_D)[lane];
        double d = static_cast<double>(qv.x) * kv.x;
        d = fma(static_cast<double>(qv.y), static_cast<double>(kv.y), d);
        d = fma(static_cast<double>(qv.z), static_cast<double>(kv.z), d);
        d = fma(static_cast<double>(qv.w), static_cast<double>(kv.w), d);
        const double s = warp_sum_f64(d) * 0.088388347648318440550;  // 128^-1/2
        if (lane == 0) e[k] = s;
        smax = fmax(smax, s);
    }
    if (lane == 0) red[warp] = smax;
    __syncthreads();
    smax = red[0];
#pragma unroll
    for (int w = 1; w < ADA_SELECT_THREADS / 32; ++w) smax = fmax(smax, red[w]);
    for (int k = tid; k < n_t; k += ADA_SELECT_THREADS) e[k] = min(ATT_BKV, p.L - k * ATT_BKV) * exp(e[k] - smax);
    __syncthreads();
    // rank of every non-forced tile in the order e descending, ties to the lower index
    for (int k = tid; k < n_t; k += ADA_SELECT_THREADS) {
        if (forced(k)) {
            rank[k] = -1;
            continue;
        }
        const double ek = e[k];
        int r = 0;
        for (int j = 0; j < n_t; ++j) r += !forced(j) && (e[j] > ek || (e[j] == ek && j < k));
        rank[k] = r;
        sorted[r] = ek;
    }
    __syncthreads();
    if (tid == 0) {
        double total = 0.0, cum = 0.0;
        int n_forced = 0;
        for (int k = 0; k < n_t; ++k) {
            total += e[k];
            if (forced(k)) { cum += e[k]; ++n_forced; }
        }
        const int n_free = n_t - n_forced;
        const int cap = p.max_tiles < 0 ? n_free : min(p.max_tiles, n_free);
        int m = 0;
        if (p.mass >= 1.0) {
            m = cap;
        } else {
            const double target = p.mass * total;
            while (m < cap && cum < target) cum += sorted[m++];
        }
        taken = m;
        p.counts[bh * n_t + q] = n_forced + m;
    }
    __syncthreads();
    const int m = taken;
    uint32_t* row = p.bits + (bh * n_t + q) * p.words;
    for (int w = warp; w < p.words; w += ADA_SELECT_THREADS / 32) {
        const int k = 32 * w + lane;
        const bool on = k < n_t && (forced(k) || rank[k] < m);
        const uint32_t word = __ballot_sync(0xffffffffu, on);
        if (lane == 0) row[w] = word;
    }
}

// One warp per (query tile, batch * head): the row's start is the sum of the counts before it (exact integer sum), and the
// bitmask expands to the ascending key tiles.
__global__ void __launch_bounds__(32) compact_tiles_kernel(const int* __restrict__ counts, const uint32_t* __restrict__ bits,
                                                           int n_t, int words, int* __restrict__ kv_tile_ptr, int64_t ptr_stride,
                                                           int* __restrict__ kv_tile_idx, int64_t idx_stride) {
    const int q = blockIdx.x, lane = threadIdx.x;
    const int64_t bh = blockIdx.y;
    const int* cnt = counts + bh * n_t;
    int start = 0;
    for (int i = lane; i < q; i += 32) start += cnt[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) start += __shfl_xor_sync(0xffffffffu, start, o);
    int* ptr = kv_tile_ptr + bh * ptr_stride;
    int* idx = kv_tile_idx + bh * idx_stride;
    if (lane == 0) {
        ptr[q + 1] = start + cnt[q];
        if (q == 0) ptr[0] = 0;
    }
    const uint32_t* row = bits + (bh * n_t + q) * words;
    for (int w = 0; w < words; ++w) {
        const uint32_t word = row[w];
        if ((word >> lane) & 1u) idx[start + __popc(word & ((1u << lane) - 1u))] = 32 * w + lane;
        start += __popc(word);
    }
}

}  // namespace scail
