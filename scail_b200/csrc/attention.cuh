// Warp-specialised flash attention forward for sm_90a (head_dim 128, bf16, non-causal).
// Replaces F.scaled_dot_product_attention in sat/transformer_defaults.py:67-72 for both the
// spatiotemporal self-attention (dit_video_crossattn_sc_xc.py:1092-1094) and the two short-KV
// cross-attention calls (:1159-1197).
//
// One CTA owns 128 query rows of one (batch, head).  Roles (12 warps = 3 warpgroups, registers re-split with setmaxnreg):
//   warpgroup 0: one TMA producer warp (Q once, K and V rings);  warpgroups 1, 2: 64 query rows each.
// Per 128-key tile a consumer warpgroup computes
//   S = Q K^T : wgmma m64n128k16 x 8, Q and K K-major from shared memory (TMA SWIZZLE_128B), S in registers,
//   online softmax on the S fragments (a row lives in the 4 lanes of a quad), P rounded to bf16 in registers,
//   O += P V  : wgmma m64n128k16 x 8 with A = P straight from registers (the S accumulator fragment IS the A-operand
//               fragment of the next MMA) and B = the V tile read MN-major from its [kv, d] layout.
// The two warpgroups run independently, so one's softmax overlaps the other's tensor-core work.
#pragma once
#include "sm90.cuh"

namespace scail {

constexpr int ATT_D = 128;
constexpr int ATT_BQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int ATT_BKV = 128;  // keys per K/V tile
constexpr int ATT_STAGES = 2;
constexpr int ATT_TILE_BYTES = 128 * 128 * 2;  // 32 KB: one 128x128 bf16 tile (two 64-column halves)
constexpr int ATT_HALF_BYTES = ATT_TILE_BYTES / 2;
constexpr int ATT_THREADS = 384;
constexpr int ATT_SMEM_BYTES = (1 + 2 * ATT_STAGES) * ATT_TILE_BYTES + 1024 + 256;
static_assert(ATT_SMEM_BYTES <= 232448, "attention: shared memory budget");

struct AttnParams {
    __nv_bfloat16* out;  // [B*q_rows_per_batch, ldo]; head h written at columns [h*128, h*128+128)
    int64_t ldo;
    int q_len;           // valid query rows per batch
    int kv_len;          // valid key rows per batch in the first key range (rows [kv_off, kv_off + kv_len) of the batch)
    int kv_off;          // first key row of range 0 inside a batch
    int kv_off1, kv_len1;  // optional second key range (kv_len1 == 0: none): context parallelism attends to "every shard but mine"
    float* o32;          // optional: write the NORMALISED partial result as fp32 [rows, ldo32] instead of bf16 `out` ...
    int64_t ldo32;
    float2* state;       // ... together with (running max in log2 units, row sum) per (row, head): [rows * H], see attn_merge_kernel
    int heads;
    int q_batch_rows;    // row stride between batches in the Q matrix / out matrix
    int kv_batch_rows;   // row stride between batches in the K/V matrices
    float scale_log2;    // softmax scale * log2(e)
    int accumulate;      // out += result (second cross-attention pass, dit_video_crossattn_sc_xc.py:1197)
};


__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                     const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t q_smem = smem_base;                                // 1 tile
    const uint32_t k_smem = smem_base + ATT_TILE_BYTES;               // ATT_STAGES tiles
    const uint32_t v_smem = k_smem + ATT_STAGES * ATT_TILE_BYTES;     // ATT_STAGES tiles
    const uint32_t bar_base = v_smem + ATT_STAGES * ATT_TILE_BYTES;
    enum {
        B_QFULL = 0,
        B_KFULL = 1,                      // [ATT_STAGES]
        B_KEMPTY = B_KFULL + ATT_STAGES,  // [ATT_STAGES]
        B_VFULL = B_KEMPTY + ATT_STAGES,  // [ATT_STAGES]
        B_VEMPTY = B_VFULL + ATT_STAGES,  // [ATT_STAGES]
        B_COUNT = B_VEMPTY + ATT_STAGES
    };
    static_assert(8 * B_COUNT <= 256, "attention: barrier area");
    auto bar = [&](int i) { return bar_base + 8u * i; };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int head = blockIdx.y;
    const int batch = blockIdx.z;
    const int q0 = blockIdx.x * ATT_BQ;
    const int n_kv0 = (p.kv_len + ATT_BKV - 1) / ATT_BKV;
    const int n_kv = n_kv0 + (p.kv_len1 + ATT_BKV - 1) / ATT_BKV;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_k);
        tma_prefetch_desc(&tmap_v);
        mbar_init(bar(B_QFULL), 1);
        for (int s = 0; s < ATT_STAGES; ++s) {
            mbar_init(bar(B_KFULL + s), 1);
            mbar_init(bar(B_KEMPTY + s), 2);  // one arrive per consumer warpgroup
            mbar_init(bar(B_VFULL + s), 1);
            mbar_init(bar(B_VEMPTY + s), 2);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            const int col = head * ATT_D;
            mbar_expect_tx(bar(B_QFULL), ATT_TILE_BYTES);
            for (int h = 0; h < 2; ++h)
                tma_load_2d(q_smem + h * ATT_HALF_BYTES, &tmap_q, bar(B_QFULL), col + h * 64, batch * p.q_batch_rows + q0);
            const int kvbase = batch * p.kv_batch_rows;
            // tile j of the concatenated key ranges starts at this row (a range's last tile may run past its end: masked)
            auto kv_row = [&](int j) { return kvbase + (j < n_kv0 ? p.kv_off + j * ATT_BKV : p.kv_off1 + (j - n_kv0) * ATT_BKV); };
            for (int j = 0; j < n_kv; ++j) {
                const int s = j % ATT_STAGES;
                const uint32_t par = ((j / ATT_STAGES) & 1) ^ 1;
                mbar_wait(bar(B_KEMPTY + s), par, 10);
                mbar_expect_tx(bar(B_KFULL + s), ATT_TILE_BYTES);
                for (int h = 0; h < 2; ++h)
                    tma_load_2d(k_smem + s * ATT_TILE_BYTES + h * ATT_HALF_BYTES, &tmap_k, bar(B_KFULL + s), col + h * 64, kv_row(j));
                mbar_wait(bar(B_VEMPTY + s), par, 11);
                mbar_expect_tx(bar(B_VFULL + s), ATT_TILE_BYTES);
                for (int h = 0; h < 2; ++h)
                    tma_load_2d(v_smem + s * ATT_TILE_BYTES + h * ATT_HALF_BYTES, &tmap_v, bar(B_VFULL + s), col + h * 64, kv_row(j));
            }
        }
    } else {
        // ===================== consumer warpgroups: QK^T, softmax, PV, epilogue =====================
        setmaxnreg_inc<232>();
        const int wg = (warp >> 2) - 1;  // rows [64 wg, 64 wg + 64) of the CTA's 128
        const int t = threadIdx.x & 127;
        const bool releaser = t == 0;
        const int quad = t & 3;
        float m_run[2] = {-INFINITY, -INFINITY};  // running max of rows r, r + 8 (already multiplied by scale_log2)
        float l_run[2] = {0.f, 0.f};               // this thread's partial row sums (reduced over the quad at the end)
        float o[ATT_D / 2];
#pragma unroll
        for (int i = 0; i < ATT_D / 2; ++i) o[i] = 0.f;
        const uint64_t q_desc = wgmma_desc_kmajor_sw128(q_smem + wg * (64 * 128));
        mbar_wait(bar(B_QFULL), 0, 20);
#pragma unroll 1
        for (int j = 0; j < n_kv; ++j) {
            const int s = j % ATT_STAGES;
            const uint32_t par = (j / ATT_STAGES) & 1;
            const int valid = j < n_kv0 ? min(ATT_BKV, p.kv_len - j * ATT_BKV) : min(ATT_BKV, p.kv_len1 - (j - n_kv0) * ATT_BKV);
            // ---- S = Q K^T ----
            float sc[ATT_BKV / 2];
            mbar_wait(bar(B_KFULL + s), par, 21);
            const uint64_t k_desc = wgmma_desc_kmajor_sw128(k_smem + s * ATT_TILE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint64_t off = ((k >> 2) * ATT_HALF_BYTES + (k & 3) * 32) >> 4;
                wgmma_ss<ATT_BKV>(sc, q_desc + off, k_desc + off, k != 0);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(sc);
            if (releaser) mbar_arrive(bar(B_KEMPTY + s));
            // ---- online softmax (thread: rows r = sc[4c + 0/1], r + 8 = sc[4c + 2/3], columns 8c + 2 quad + 0/1) ----
            if (valid < ATT_BKV) {
#pragma unroll
                for (int c = 0; c < ATT_BKV / 8; ++c) {
                    const int col = 8 * c + 2 * quad;
                    if (col >= valid) { sc[4 * c] = -INFINITY; sc[4 * c + 2] = -INFINITY; }
                    if (col + 1 >= valid) { sc[4 * c + 1] = -INFINITY; sc[4 * c + 3] = -INFINITY; }
                }
            }
            float alpha[2], neg_m[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx = -INFINITY;
#pragma unroll
                for (int c = 0; c < ATT_BKV / 8; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * h], sc[4 * c + 2 * h + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[h], mx * p.scale_log2);
                alpha[h] = fast_exp2(m_run[h] - m_new);  // 0 on the first tile (m_run = -inf)
                m_run[h] = m_new;
                l_run[h] *= alpha[h];
                neg_m[h] = -m_new;
            }
#pragma unroll
            for (int c = 0; c < ATT_D / 8; ++c) {
                o[4 * c] *= alpha[0];
                o[4 * c + 1] *= alpha[0];
                o[4 * c + 2] *= alpha[1];
                o[4 * c + 3] *= alpha[1];
            }
            uint32_t pa[ATT_BKV / 16][4];  // P as bf16 A fragments, one set of 4 registers per 16-key MMA step
#pragma unroll
            for (int c = 0; c < ATT_BKV / 8; ++c) {
                float e[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    e[i] = fast_exp2(fmaf(sc[4 * c + i], p.scale_log2, neg_m[i >> 1]));
                    l_run[i >> 1] += e[i];
                }
                pa[c >> 1][(c & 1) * 2] = pack_bf16(e[0], e[1]);
                pa[c >> 1][(c & 1) * 2 + 1] = pack_bf16(e[2], e[3]);
            }
            // ---- O += P V ----
            mbar_wait(bar(B_VFULL + s), par, 22);
            const uint64_t v_desc = wgmma_desc_mnmajor_sw128(v_smem + s * ATT_TILE_BYTES, ATT_HALF_BYTES);
            fence_regs(o);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < ATT_BKV / 16; ++k) wgmma_rs_tb<ATT_D>(o, pa[k], v_desc + k * (2048 >> 4));  // 16 kv rows = 2048 B
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
            if (releaser) mbar_arrive(bar(B_VEMPTY + s));
        }
        // ---- epilogue: O / l -> bf16 (or normalised fp32 partial + (m, l)) -> global ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
            l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int qi = q0 + wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + 8 * h;
            if (qi >= p.q_len) continue;
            const float inv_l = 1.0f / l_run[h];
            const int64_t grow = static_cast<int64_t>(batch) * p.q_batch_rows + qi;
            if (p.o32 != nullptr) {  // partial result over a subset of the keys: fp32, merged later (attn_merge_kernel)
                if (quad == 0) p.state[grow * p.heads + head] = make_float2(m_run[h], l_run[h]);
                float* dst = p.o32 + grow * p.ldo32 + head * ATT_D + 2 * quad;
#pragma unroll
                for (int c = 0; c < ATT_D / 8; ++c)
                    *reinterpret_cast<float2*>(dst + 8 * c) = make_float2(o[4 * c + 2 * h] * inv_l, o[4 * c + 2 * h + 1] * inv_l);
                continue;
            }
            __nv_bfloat16* dst = p.out + grow * p.ldo + head * ATT_D + 2 * quad;
#pragma unroll
            for (int c = 0; c < ATT_D / 8; ++c) {
                float f0 = o[4 * c + 2 * h] * inv_l, f1 = o[4 * c + 2 * h + 1] * inv_l;
                uint32_t* d32 = reinterpret_cast<uint32_t*>(dst + 8 * c);
                if (p.accumulate) {
                    const float2 prev = unpack_bf16(*d32);
                    f0 += prev.x;
                    f1 += prev.y;
                }
                *d32 = pack_bf16(f0, f1);
            }
        }
    }
}

// Combine two partial attention results over disjoint key sets (context parallelism: local shard first, remote shards once
// the all-gather has landed).  Each partial is normalised by its own row sum l and carries (m, l) with m in log2 units:
//   out = (w_a O_a + w_b O_b) / (w_a + w_b),  w_x = l_x 2^(m_x - max(m_a, m_b)).   One warp per (row, head).
__global__ void __launch_bounds__(256) attn_merge_kernel(const float* __restrict__ oa, const float2* __restrict__ sa,
                                                         const float* __restrict__ ob, const float2* __restrict__ sb,
                                                         __nv_bfloat16* __restrict__ out, int64_t ld32, int64_t ldo, int64_t rows,
                                                         int heads) {
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;  // (row, head)
    if (item >= rows * heads) return;
    const int lane = threadIdx.x & 31;
    const int64_t row = item / heads;
    const int head = static_cast<int>(item - row * heads);
    const float2 a = sa[item], b = sb[item];
    const float m = fmaxf(a.x, b.x);
    const float wa = a.y * fast_exp2(a.x - m), wb = b.y * fast_exp2(b.x - m);
    const float inv = 1.0f / (wa + wb);
    const float ca = wa * inv, cb = wb * inv;
    const float4 va = *reinterpret_cast<const float4*>(oa + row * ld32 + head * ATT_D + lane * 4);
    const float4 vb = *reinterpret_cast<const float4*>(ob + row * ld32 + head * ATT_D + lane * 4);
    uint2 o;
    o.x = pack_bf16(ca * va.x + cb * vb.x, ca * va.y + cb * vb.y);
    o.y = pack_bf16(ca * va.z + cb * vb.z, ca * va.w + cb * vb.w);
    *reinterpret_cast<uint2*>(out + row * ldo + head * ATT_D + lane * 4) = o;
}

}  // namespace scail
