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
// The two warpgroups take strict turns at the tensor cores (named barriers 1 and 2): a turn issues PV of the previous tile
// and QK^T of the next, so one warpgroup's softmax always runs under the other's MMAs.
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
constexpr int ATT_TURN_BAR = 1;  // named barriers 1 and 2: the consumer warpgroups' MMA turns (attention_fwd_kernel)
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
    const int* kv_tile_ptr;  // block-sparse map (attention_fwd_kernel<true> only, one range, kv_off = 0): query tile t attends
    const int* kv_tile_idx;  // the key tiles kv_tile_idx[kv_tile_ptr[t] .. kv_tile_ptr[t + 1]), strictly ascending
    int64_t ptr_stride;      // per-(batch, head) maps: (b, h) reads kv_tile_ptr + (b H + h) ptr_stride and kv_tile_idx +
    int64_t idx_stride;      // (b H + h) idx_stride; both 0: one map serves every (batch, head)
};


// kSparse: the CTA's key tiles are the row blockIdx.x of the block-sparse map (AttnParams::kv_tile_ptr / kv_tile_idx; with
// non-zero strides, the map of the CTA's own (batch, head)) instead of every tile of the key ranges.  Only the tile list changes: tile j of the row is loaded from key row 128 kv_tile_idx[j],
// its valid-key mask is taken from that global start, and the turns run over the row's n_kv tiles exactly as below.
template <bool kSparse>
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
    const int64_t bh_map = kSparse ? static_cast<int64_t>(batch) * p.heads + head : 0;  // this (b, h)'s map
    const int* tile_ptr = kSparse ? p.kv_tile_ptr + bh_map * p.ptr_stride : nullptr;
    const int* kv_tiles = kSparse ? p.kv_tile_idx + bh_map * p.idx_stride + tile_ptr[blockIdx.x] : nullptr;
    const int n_kv0 = kSparse ? tile_ptr[blockIdx.x + 1] - tile_ptr[blockIdx.x] : (p.kv_len + ATT_BKV - 1) / ATT_BKV;
    const int n_kv = kSparse ? n_kv0 : n_kv0 + (p.kv_len1 + ATT_BKV - 1) / ATT_BKV;

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
            auto kv_row = [&](int j) {
                if (kSparse) return kvbase + p.kv_off + kv_tiles[j] * ATT_BKV;
                return kvbase + (j < n_kv0 ? p.kv_off + j * ATT_BKV : p.kv_off1 + (j - n_kv0) * ATT_BKV);
            };
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
        uint32_t pa[ATT_BKV / 16][4];  // P of the last softmaxed tile as bf16 A fragments, one set per 16-key MMA step
        const uint64_t q_desc = wgmma_desc_kmajor_sw128(q_smem + wg * (64 * 128));
        mbar_wait(bar(B_QFULL), 0, 20);
        // S = Q K^T of tile j into sc (issued and committed, not waited for)
        auto issue_qk = [&](int j, float(&sc)[ATT_BKV / 2]) {
            const uint64_t k_desc = wgmma_desc_kmajor_sw128(k_smem + (j % ATT_STAGES) * ATT_TILE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint64_t off = ((k >> 2) * ATT_HALF_BYTES + (k & 3) * 32) >> 4;
                wgmma_ss<ATT_BKV>(sc, q_desc + off, k_desc + off, k != 0);
            }
            wgmma_commit();
        };
        // O += P V of tile j, waited for; the V stage is released
        auto pv = [&](int j) {
            const int s = j % ATT_STAGES;
            const uint64_t v_desc = wgmma_desc_mnmajor_sw128(v_smem + s * ATT_TILE_BYTES, ATT_HALF_BYTES);
            fence_regs(o);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < ATT_BKV / 16; ++k) wgmma_rs_tb<ATT_D>(o, pa[k], v_desc + k * (2048 >> 4));  // 16 kv rows = 2048 B
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
            if (releaser) mbar_arrive(bar(B_VEMPTY + s));
        };
        // waits for S of tile j, releases the K stage, then the online softmax: O *= alpha, P -> pa
        // (thread: rows r = sc[4c + 0/1], r + 8 = sc[4c + 2/3], columns 8c + 2 quad + 0/1)
        auto softmax = [&](int j, float(&sc)[ATT_BKV / 2]) {
            const int valid = kSparse    ? min(ATT_BKV, p.kv_len - kv_tiles[j] * ATT_BKV)
                              : j < n_kv0 ? min(ATT_BKV, p.kv_len - j * ATT_BKV)
                                          : min(ATT_BKV, p.kv_len1 - (j - n_kv0) * ATT_BKV);
            wgmma_wait<0>();
            fence_regs(sc);
            if (releaser) mbar_arrive(bar(B_KEMPTY + j % ATT_STAGES));
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
        };
        // Ping-pong: the two warpgroups take turns at the tensor cores.  Turn j of a warpgroup issues O += P V of tile j - 1,
        // waits for it, issues S = Q K^T of tile j and passes the turn on; the softmax of tile j then runs while the other
        // warpgroup's turn keeps the tensor cores busy.  Named barrier ATT_TURN_BAR + w is warpgroup w's turn: w waits on it
        // (bar.sync) and the other warpgroup arrives on it (bar.arrive) when its own turn ends.  Warpgroup 0 takes turn 0
        // without waiting and warpgroup 1's last turn passes nothing on, so both take n_kv + 1 turns (whether or not their
        // rows are valid), every barrier phase sees exactly 256 threads and none is left pending at exit.  The host requires
        // kv_len > 0, so n_kv >= 1.  The first and last turns are peeled rather than guarded inside one loop: a wgmma under
        // a branch makes ptxas serialise all of them (C7518).  PV is waited for before QK^T is issued, so P (32 registers)
        // and S (64) are never live together beside O (64): the schedule fits the 168 registers of the 384-thread bound.
        const int turn_bar = ATT_TURN_BAR + wg, next_bar = ATT_TURN_BAR + (wg ^ 1);
        {
            float sc[ATT_BKV / 2];
            mbar_wait(bar(B_KFULL), 0, 21);
            if (wg == 1) named_bar_sync(turn_bar, 256);
            issue_qk(0, sc);
            named_bar_arrive(next_bar, 256);
            softmax(0, sc);
        }
#pragma unroll 1
        for (int j = 1; j < n_kv; ++j) {
            float sc[ATT_BKV / 2];
            mbar_wait(bar(B_KFULL + j % ATT_STAGES), (j / ATT_STAGES) & 1, 21);
            mbar_wait(bar(B_VFULL + (j - 1) % ATT_STAGES), ((j - 1) / ATT_STAGES) & 1, 22);
            named_bar_sync(turn_bar, 256);
            pv(j - 1);
            issue_qk(j, sc);
            named_bar_arrive(next_bar, 256);
            softmax(j, sc);
        }
        mbar_wait(bar(B_VFULL + (n_kv - 1) % ATT_STAGES), ((n_kv - 1) / ATT_STAGES) & 1, 22);
        named_bar_sync(turn_bar, 256);
        pv(n_kv - 1);
        if (wg == 0) named_bar_arrive(next_bar, 256);
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

// ================================================================================================================
// FP8 (e4m3) self-attention (q_len == kv_len == L), opt-in.  Operands, as rmsnorm_rope_kernel<true> and quant_vt_fp8_kernel
// write them (the e4m3 row format of rowops.cuh: s = amax / 448, q = satfinite_rn(x / s), s = 1 for a zero row):
//   Q, K : e4m3 [B*L, ld] (head h = columns h*128..), one fp32 scale per (token, head): head-major [B, H, L_pad]
//   V^T  : e4m3 [B, H, 128, L_pad] (keys contiguous, permuted inside every 16-key group by fp8_vt_key, zero past L),
//          one fp32 scale per (batch, head, channel) over all L keys: [B, H, 128]
//   P    : fixed scale, P^ = e4m3(2^8 * exp2(s - m_running)); the 2^8 is the +8 in the exp2 argument.  l sums the fp32 values.
// Same roles as attention_fwd_kernel: a TMA producer warp and two consumer warpgroups of 64 query rows; one CTA per 128
// query rows of one (batch, head).  Every Q / K / V^T tile is one 128 x 128-byte SWIZZLE_128B box (16 KB).
//   S = Q K^T : wgmma m64n128k32 e4m3 x 4 (descriptor +2 per k32 step); S *= K scale per column, then the bf16 kernel's
//               online softmax with the row's Q scale folded into scale_log2.
//   O_t = P^ V^ : wgmma m64n128k32 x 4 with A = P^ from registers into a fresh accumulator (Hopper's fp8 wgmma keeps ~14
//               accumulator bits), then O = O * alpha + O_t in fp32.
// P^ as the A operand without shuffles: a thread holds S columns {2q, 2q+1, 8+2q, 9+2q, ...} of each 32-key group but the
// A fragment wants k = 4q..4q+3 (wgmma_rs_e4m3).  So the reduction is reindexed instead of the data: register a[0] of key
// group g packs S columns 32g + {2q, 2q+1, 8+2q, 9+2q}, and V^T column k holds key fp8_vt_key(k), the inverse relabelling.
constexpr int ATT8_STAGES = 4;
constexpr int ATT8_TILE_BYTES = 128 * 128;  // 16 KB: one e4m3 tile
constexpr int ATT8_KS_BYTES = ATT_BKV * 4;  // the K tile's 128 fp32 scales
constexpr int ATT8_SMEM_BYTES = (1 + 2 * ATT8_STAGES) * ATT8_TILE_BYTES + ATT8_STAGES * ATT8_KS_BYTES + 1024 + 256;
static_assert(ATT8_SMEM_BYTES <= 232448, "attention_fp8: shared memory budget");

// the key stored at logical column k of V^T (a permutation inside every 16-key group)
__host__ __device__ __forceinline__ int fp8_vt_key(int k) {
    return 16 * (k / 16) + 2 * ((k % 16) / 4) + (k % 2) + 8 * ((k % 4) / 2);
}

struct Attn8Params {
    __nv_bfloat16* out;  // [B*L, ldo] bf16, head h at columns [h*128, h*128+128)
    int64_t ldo;
    const float* q_scale;   // [B, H, L_pad]
    const float* k_scale;   // [B, H, L_pad]
    const float* v_scale;   // [B, H, 128]
    int L, L_pad, heads;
    float scale_log2;       // softmax scale * log2(e)
    const int* kv_tile_ptr;  // block-sparse map (attention_fp8_kernel<true> only), as AttnParams
    const int* kv_tile_idx;
    int64_t ptr_stride, idx_stride;  // per-(batch, head) maps, as AttnParams (0: shared)
};

// kSparse: the block-sparse map selects the CTA's key tiles, as in attention_fwd_kernel<true>; tile j's K rows, K scales
// and V^T columns start at key 128 kv_tile_idx[j].
// kInt8QK (fp8_attention="int8_qk"): Q and K are INT8 codes in [-127, 127] with the same per-(token, head) scales (the INT8
// row format of rowops.cuh; K smoothed by its per-(batch, channel) mean first, quant_k_int8), and S = Q K^T runs as
// wgmma m64n128k32 s8 x 4 into s32.  V^, P^ and everything after S are unchanged.  Subtracting k-bar from every key shifts
// each logit of a query row by the same q . k-bar, which the softmax cancels, so the listed tiles of a sparse map need no
// correction either.
template <bool kSparse, bool kInt8QK = false>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                     const __grid_constant__ CUtensorMap tmap_vt, const Attn8Params p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t q_smem = smem_base;
    const uint32_t k_smem = q_smem + ATT8_TILE_BYTES;
    const uint32_t v_smem = k_smem + ATT8_STAGES * ATT8_TILE_BYTES;
    const uint32_t ks_smem = v_smem + ATT8_STAGES * ATT8_TILE_BYTES;
    const uint32_t bar_base = ks_smem + ATT8_STAGES * ATT8_KS_BYTES;
    enum {
        B_QFULL = 0,
        B_KFULL = 1,
        B_KEMPTY = B_KFULL + ATT8_STAGES,
        B_VFULL = B_KEMPTY + ATT8_STAGES,
        B_VEMPTY = B_VFULL + ATT8_STAGES,
        B_COUNT = B_VEMPTY + ATT8_STAGES
    };
    static_assert(8 * B_COUNT <= 256, "attention_fp8: barrier area");
    auto bar = [&](int i) { return bar_base + 8u * i; };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int head = blockIdx.y;
    const int batch = blockIdx.z;
    const int q0 = blockIdx.x * ATT_BQ;
    const int64_t bh = static_cast<int64_t>(batch) * p.heads + head;
    const int* tile_ptr = kSparse ? p.kv_tile_ptr + bh * p.ptr_stride : nullptr;  // this (b, h)'s map
    const int* kv_tiles = kSparse ? p.kv_tile_idx + bh * p.idx_stride + tile_ptr[blockIdx.x] : nullptr;
    const int n_kv = kSparse ? tile_ptr[blockIdx.x + 1] - tile_ptr[blockIdx.x] : (p.L + ATT_BKV - 1) / ATT_BKV;
    auto kv_start = [&](int j) { return (kSparse ? kv_tiles[j] : j) * ATT_BKV; };  // first key of the CTA's tile j

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_k);
        tma_prefetch_desc(&tmap_vt);
        mbar_init(bar(B_QFULL), 1);
        for (int s = 0; s < ATT8_STAGES; ++s) {
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
            const int row0 = batch * p.L;
            mbar_expect_tx(bar(B_QFULL), ATT8_TILE_BYTES);
            tma_load_2d(q_smem, &tmap_q, bar(B_QFULL), col, row0 + q0);
            const float* ks = p.k_scale + bh * p.L_pad;
            for (int j = 0; j < n_kv; ++j) {
                const int s = j % ATT8_STAGES;
                const uint32_t par = ((j / ATT8_STAGES) & 1) ^ 1;
                mbar_wait(bar(B_KEMPTY + s), par, 10);
                mbar_expect_tx(bar(B_KFULL + s), ATT8_TILE_BYTES + ATT8_KS_BYTES);
                const int k0 = kv_start(j);
                tma_load_2d(k_smem + s * ATT8_TILE_BYTES, &tmap_k, bar(B_KFULL + s), col, row0 + k0);
                bulk_load_1d(ks_smem + s * ATT8_KS_BYTES, ks + k0, ATT8_KS_BYTES, bar(B_KFULL + s));
                mbar_wait(bar(B_VEMPTY + s), par, 11);
                mbar_expect_tx(bar(B_VFULL + s), ATT8_TILE_BYTES);
                tma_load_2d(v_smem + s * ATT8_TILE_BYTES, &tmap_vt, bar(B_VFULL + s), k0, static_cast<int>(bh * ATT_D));
            }
        }
    } else {
        // ===================== consumer warpgroups =====================
        setmaxnreg_inc<232>();
        const int wg = (warp >> 2) - 1;
        const int t = threadIdx.x & 127;
        const bool releaser = t == 0;
        const int quad = t & 3;
        const int r0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);  // rows r0, r0 + 8 of the CTA's 128
        float sl2[2];  // scale_log2 * Q scale of the two rows (rows past L read the zero-filled padding: masked at the end)
#pragma unroll
        for (int h = 0; h < 2; ++h) sl2[h] = p.scale_log2 * p.q_scale[bh * p.L_pad + q0 + r0 + 8 * h];
        float m_run[2] = {-INFINITY, -INFINITY};
        float l_run[2] = {0.f, 0.f};
        float o[ATT_D / 2];
#pragma unroll
        for (int i = 0; i < ATT_D / 2; ++i) o[i] = 0.f;
        const uint64_t q_desc = wgmma_desc_kmajor_sw128(q_smem + wg * (64 * 128));
        mbar_wait(bar(B_QFULL), 0, 20);
#pragma unroll 1
        for (int j = 0; j < n_kv; ++j) {
            const int s = j % ATT8_STAGES;
            const uint32_t par = (j / ATT8_STAGES) & 1;
            const int valid = min(ATT_BKV, p.L - kv_start(j));
            // ---- S = Q K^T ----
            float sc[ATT_BKV / 2];
            mbar_wait(bar(B_KFULL + s), par, 21);
            const uint64_t k_desc = wgmma_desc_kmajor_sw128(k_smem + s * ATT8_TILE_BYTES);
            if constexpr (kInt8QK) {
                // s32 accumulator started at the bits of 1.5 * 2^23: |S| < 2^22 keeps the sum inside [2^23, 2^24), where the
                // bits read as the float 1.5 * 2^23 + S exactly, so one exact FADD converts it (no I2F)
                uint32_t si[ATT_BKV / 2];
#pragma unroll
                for (int i = 0; i < ATT_BKV / 2; ++i) si[i] = 0x4B400000u;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_ss_s8<ATT_BKV>(si, q_desc + 2 * k, k_desc + 2 * k);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(si);
#pragma unroll
                for (int i = 0; i < ATT_BKV / 2; ++i) sc[i] = __fsub_rn(__uint_as_float(si[i]), 12582912.0f);
            } else {
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_ss_e4m3<ATT_BKV>(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(sc);
            }
            // K scales of this thread's columns 8c + 2 quad + {0, 1}
            const uint32_t ksa = ks_smem + s * ATT8_KS_BYTES + 8 * quad;
#pragma unroll
            for (int c = 0; c < ATT_BKV / 8; ++c) {
                const float2 ksc = lds_f2(ksa + 32 * c);
                sc[4 * c] *= ksc.x;
                sc[4 * c + 1] *= ksc.y;
                sc[4 * c + 2] *= ksc.x;
                sc[4 * c + 3] *= ksc.y;
            }
            if (releaser) mbar_arrive(bar(B_KEMPTY + s));
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
                const float m_new = fmaxf(m_run[h], mx * sl2[h]);  // sl2 > 0: the max commutes with the scaling
                alpha[h] = fast_exp2(m_run[h] - m_new);
                m_run[h] = m_new;
                l_run[h] *= alpha[h];
                neg_m[h] = 8.0f - m_new;  // P^ = 2^8 exp2(s - m)
            }
            // P^ as e4m3 A fragments, one set of 4 registers per 32-key group g: a[0] = row r0, S columns 32g + {2q, 2q+1,
            // 8+2q, 9+2q} = sc[16g + {0, 1, 4, 5}]; a[1] = row r0 + 8 (sc[16g + {2, 3, 6, 7}]); a[2], a[3]: the same + 8 sc
            uint32_t pa[ATT_BKV / 32][4];
#pragma unroll
            for (int g = 0; g < ATT_BKV / 32; ++g) {
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int b0 = 16 * g + 8 * (r >> 1) + 2 * (r & 1);  // sc index of the first of the four values
                    const int h = r & 1;
                    float e[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        e[i] = fast_exp2(fmaf(sc[b0 + (i & 1) + 4 * (i >> 1)], sl2[h], neg_m[h]));
                        l_run[h] += e[i];
                    }
                    pa[g][r] = pack_e4m3x4(e[0], e[1], e[2], e[3]);
                }
            }
            // ---- O_t = P^ V^ (fresh accumulator), O = O * alpha + O_t ----
            float ot[ATT_D / 2];
            mbar_wait(bar(B_VFULL + s), par, 22);
            const uint64_t v_desc = wgmma_desc_kmajor_sw128(v_smem + s * ATT8_TILE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int g = 0; g < ATT_BKV / 32; ++g) wgmma_rs_e4m3<ATT_D>(ot, pa[g], v_desc + 2 * g, g != 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(ot);
            if (releaser) mbar_arrive(bar(B_VEMPTY + s));
#pragma unroll
            for (int c = 0; c < ATT_D / 8; ++c) {
                o[4 * c] = fmaf(o[4 * c], alpha[0], ot[4 * c]);
                o[4 * c + 1] = fmaf(o[4 * c + 1], alpha[0], ot[4 * c + 1]);
                o[4 * c + 2] = fmaf(o[4 * c + 2], alpha[1], ot[4 * c + 2]);
                o[4 * c + 3] = fmaf(o[4 * c + 3], alpha[1], ot[4 * c + 3]);
            }
        }
        // ---- epilogue: O * s_v[channel] / l -> bf16 ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
            l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
        }
        const float* vs = p.v_scale + bh * ATT_D + 2 * quad;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int qi = q0 + r0 + 8 * h;
            if (qi >= p.L) continue;
            const float inv_l = 1.0f / l_run[h];
            __nv_bfloat16* dst = p.out + (static_cast<int64_t>(batch) * p.L + qi) * p.ldo + head * ATT_D + 2 * quad;
#pragma unroll
            for (int c = 0; c < ATT_D / 8; ++c) {
                const float2 sv = *reinterpret_cast<const float2*>(vs + 8 * c);
                *reinterpret_cast<uint32_t*>(dst + 8 * c) =
                    pack_bf16(o[4 * c + 2 * h] * sv.x * inv_l, o[4 * c + 2 * h + 1] * sv.y * inv_l);
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
