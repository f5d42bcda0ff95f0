// Fused multi-head self-attention on the Hopper tensor cores (wgmma + TMA + mbarrier), head dim 64, bf16:
//     O = dropout(softmax((Q / sqrt(d)) K^T)) V            (reference: trainer/model/modules/multi_headed_attn.py:199-223)
// and its backward, without ever writing the [B, heads, T, T] score / probability tensors to HBM.
//
// One CTA = 128 "stationary" rows of one (batch, head) x all 64-row "streamed" tiles of the other operand:
//   MODE 0  forward          stationary = queries   S = Q K^T -> P -> O += P V ;  writes O and the row log-sum-exp
//   MODE 1  backward, dQ     stationary = queries   recomputes P, dP = dO V^T, dS = P o (dP - D), dQ += dS K
//   MODE 2  backward, dK/dV  stationary = keys      works on S^T: dV += P^T dO, dK += dS^T Q
// (every output row has one owner: no atomics, bit-reproducible).
//
// Warp roles (384 threads):
//   warpgroup 0      TMA loader (one converged warp): stationary tiles once, streamed tiles (and, in MODE 2, the per-query lse / D
//                    vectors) through a TA_NST-stage mbarrier ring
//   warpgroups 1, 2  consumers, 64 stationary rows each: S (and dP) = A_stat X^T with wgmma from shared memory, fp32 in registers;
//                    softmax / dropout / dS in registers; the bf16 result feeds the second product (acc (+)= P X) straight from
//                    registers (the accumulator layout of an m64 x 16 block is the A-operand layout of wgmma).
//
// Dropout: counter-based mask shared with the stand-alone softmax kernels -- one 32-bit hash per PAIR of adjacent keys
// (index (row * ceil(T/2) + key/2) over the [B*heads*T, T] probability matrix), 16 bits per element.  The kernels are compiled
// per dropout case (template DROP): none, hashed from the seed in every mode (pk_attention_fwd / _bwd), or keep bits
// (pk_attention_fwd_bits / _bwd_bits): the forward alone hashes and writes each decision as one bit (layout in
// include/pika_b200.h), and the backward reads them -- MODE 1 one word per thread and tile straight from global memory, MODE 2 the
// transposed 64 x 128 block through the loader's ring.
//
// Chunk mask (template CHUNK; pk_attention_fwd_chunk / _bwd_chunk, DESIGN.md "Chunked attention"): frame t lies in chunk
// (t + chunk_off) / chunk_len, and query i sees key j iff chunk(i) - left_chunks <= chunk(j) <= chunk(i) (left_chunks = -1: no lower
// limit).  A row's allowed streamed indices form one interval whose ends never decrease with the row, so a CTA streams only the tiles
// between the first row's lower end and the last row's upper end (the loader and both consumer warpgroups derive the same trip
// count from the same rows), and the per-element mask runs only on tiles that some row of the warpgroup does not see whole.
#include <cstdlib>
#include <cstring>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

constexpr int TA_BR = 128;
constexpr int TA_BC = 64;
constexpr int TA_NST = 4;
constexpr int TA_THREADS = 384;
constexpr float TA_LOG2E = 1.4426950408889634f;
constexpr float TA_LN2 = 0.6931471805599453f;

constexpr int TA_TILE_S = TA_BR * 128;            // 16 KB: 128 rows x 64 bf16
constexpr int TA_TILE_X = TA_BC * 128;            // 8 KB
constexpr int TA_OFF_STAT = 0;                    // two stationary tiles
constexpr int TA_OFF_RING = 2 * TA_TILE_S;        // NST x (X1, X2)
constexpr int TA_OFF_VEC = TA_OFF_RING + TA_NST * 2 * TA_TILE_X;       // [NST][2][64] floats (MODE 2: lse, D of the streamed queries)
enum : int { TA_DROP_NONE = 0, TA_DROP_HASH = 1, TA_DROP_BITS = 2 };
constexpr int TA_KB_BLOCK = 512;                                        // keep bits of one 64 x 64 (query, key) block
constexpr int TA_OFF_KB = TA_OFF_VEC + TA_NST * 2 * TA_BC * 4;          // [NST][2 blocks] keep bits (MODE 2, dropout)
constexpr int TA_OFF_BAR = TA_OFF_KB + TA_NST * 2 * TA_KB_BLOCK;
constexpr int TA_SMEM = TA_OFF_BAR + 256 + 1024;

struct AttnTcParams {
    CUtensorMap q, k, v, dout;                    // [B][T][heads*64] bf16, box 64 x 64 x 1, 128B swizzle
    __nv_bfloat16* out; long long ld_o;
    __nv_bfloat16* dq; __nv_bfloat16* dk; __nv_bfloat16* dv; long long ld_dqkv;
    float* lse;                                   // [B*heads][Tpad] natural-log row log-sum-exp of the scaled scores
    float* dsum;                                  // [B*heads][Tpad] D_i = sum_d dO_id O_id
    uint32_t* keep_bits;                          // [B*heads][nkb][nkb][128] words (MODE 0 writes, MODES 1 / 2 read); dropout only
    int B, T, heads, Tpad, Tp2, nkb;
    float alpha;
    uint32_t thresh16; float drop_scale; uint32_t seed;
    int chunk_len, chunk_off, left_chunks;        // CHUNK only
};

// stationary row -> its allowed streamed interval in MODE (0 / 1: keys of a query, 2: queries of a key)
template <int MODE> PK_DEVICE int chunk_lo(const AttnTcParams& p, int r) {
    return MODE == 2 ? chunk_query_lo(r, p.T, p.chunk_len, p.chunk_off) : chunk_key_lo(r, p.T, p.chunk_len, p.chunk_off, p.left_chunks);
}
template <int MODE> PK_DEVICE int chunk_hi(const AttnTcParams& p, int r) {
    return MODE == 2 ? chunk_query_hi(r, p.T, p.chunk_len, p.chunk_off, p.left_chunks) : chunk_key_hi(r, p.T, p.chunk_len, p.chunk_off);
}
// the 64-wide streamed tiles [jb, je) that stationary rows [row_base, row_base + 128) of the CTA visit; never empty (a frame sees itself)
template <int MODE> PK_DEVICE void chunk_tiles(const AttnTcParams& p, int row_base, int& jb, int& je) {
    jb = chunk_lo<MODE>(p, row_base) / TA_BC;
    je = (chunk_hi<MODE>(p, min(row_base + TA_BR, p.T) - 1) + TA_BC - 1) / TA_BC;
}

// A-operand fragment k-block kk (16 streamed indices) of a 64 x 64 register tile
PK_DEVICE void frag_a(const float (&x)[32], int kk, uint32_t (&a)[4]) {
    a[0] = pack_bf16x2(x[8 * kk + 0], x[8 * kk + 1]);
    a[1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
    a[2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]);
    a[3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
}
// first word of the keep bits of query block qb x key block kb (64 x 64 each) of (batch, head) bh
PK_DEVICE size_t kb_block(const AttnTcParams& p, int bh, int qb, int kb) { return (((size_t)bh * p.nkb + qb) * p.nkb + kb) * (TA_KB_BLOCK / 4); }
PK_DEVICE float quad_max(float v) { return fmaxf(v, fmaxf(__shfl_xor_sync(0xffffffffu, v, 1), __shfl_xor_sync(0xffffffffu, fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1)), 2))); }
PK_DEVICE float quad_sum(float v) { v += __shfl_xor_sync(0xffffffffu, v, 1); return v + __shfl_xor_sync(0xffffffffu, v, 2); }

// stores a 64 x 64 fp32 register tile (rows >= T skipped) as bf16, scaled
PK_DEVICE void store_tile(const float (&x)[32], __nv_bfloat16* base, long long ld, int row0, int T, int r0, int cq, float sc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = row0 + r0 + 8 * h;
        if (row >= T) continue;
        __nv_bfloat16* orow = base + (long long)row * ld;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
            *reinterpret_cast<uint32_t*>(orow + nb * 8 + cq) = pack_bf16x2(x[nb * 4 + 2 * h] * sc, x[nb * 4 + 2 * h + 1] * sc);
    }
}

// DROP: TA_DROP_NONE (p = 0: no mask code at all), TA_DROP_HASH (every mode hashes the mask from the seed) or TA_DROP_BITS (MODE 0
// hashes it and writes the keep bits, MODES 1 / 2 read them)
template <int MODE, int DROP, bool CHUNK = false>
__global__ void __launch_bounds__(TA_THREADS, 1) attention_tc_kernel(const __grid_constant__ AttnTcParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TA_OFF_BAR);
    uint64_t* stat_full = bars;               // 1
    uint64_t* full_bar = bars + 1;            // NST
    uint64_t* empty_bar = full_bar + TA_NST;  // NST
    float* vec = reinterpret_cast<float*>(smem + TA_OFF_VEC);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int T = p.T;
    const int bh = blockIdx.y, b = bh / p.heads, h = bh - b * p.heads;
    const int row_base = blockIdx.x * TA_BR;
    int j_begin = 0, j_end = (T + TA_BC - 1) / TA_BC;
    if (CHUNK) chunk_tiles<MODE>(p, row_base, j_begin, j_end);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.q); tma_prefetch_desc(&p.k); tma_prefetch_desc(&p.v);
        if (MODE != 0) tma_prefetch_desc(&p.dout);
        mbar_init(stat_full, 1);
        for (int s = 0; s < TA_NST; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp != 0) return;
        // ===================================================== TMA loader (converged warp, one elected lane issues)
        const uint32_t lead = elect_one_u32();
        const CUtensorMap* ma0 = (MODE == 2) ? &p.k : &p.q;
        const CUtensorMap* ma1 = (MODE == 2) ? &p.v : &p.dout;
        const CUtensorMap* mx1 = (MODE == 2) ? &p.q : &p.k;
        const CUtensorMap* mx2 = (MODE == 2) ? &p.dout : &p.v;
        mbar_arrive_expect_tx_p(stat_full, (MODE == 0 ? 1 : 2) * TA_TILE_S, lead);
        for (int half = 0; half < 2; ++half) {
            tma_load_3d_p(smem + TA_OFF_STAT + half * TA_TILE_X, ma0, stat_full, h * 64, row_base + half * 64, b, lead);
            if (MODE != 0) tma_load_3d_p(smem + TA_OFF_STAT + TA_TILE_S + half * TA_TILE_X, ma1, stat_full, h * 64, row_base + half * 64, b, lead);
        }
        constexpr bool kb_load = MODE == 2 && DROP == TA_DROP_BITS;
        int stage = 0;
        uint32_t phase = 0;
        for (int j = j_begin; j < j_end; ++j) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* x1 = smem + TA_OFF_RING + stage * 2 * TA_TILE_X;
            // CHUNK: the forward wrote the keep bits of key block 2 * blockIdx.x + half for query tile j only if the forward CTA of
            // query rows [(j / 2) * 128, +128) visited it; a block it skipped is not read (every pair of it is masked)
            bool kb_half[2] = {kb_load, kb_load};
            if (CHUNK && kb_load) {
                int qb, qe;
                chunk_tiles<0>(p, (j >> 1) * TA_BR, qb, qe);
                kb_half[0] = 2 * (int)blockIdx.x >= qb && 2 * (int)blockIdx.x < qe;
                kb_half[1] = 2 * (int)blockIdx.x + 1 >= qb && 2 * (int)blockIdx.x + 1 < qe;
            }
            mbar_arrive_expect_tx_p(&full_bar[stage], 2 * TA_TILE_X + (MODE == 2 ? 2 * TA_BC * 4 : 0) + ((int)kb_half[0] + (int)kb_half[1]) * TA_KB_BLOCK,
                                    lead);
            tma_load_3d_p(x1, mx1, &full_bar[stage], h * 64, j * TA_BC, b, lead);
            tma_load_3d_p(x1 + TA_TILE_X, mx2, &full_bar[stage], h * 64, j * TA_BC, b, lead);
            if (MODE == 2) {
                const size_t off = (size_t)bh * p.Tpad + (size_t)j * TA_BC;
                bulk_load_p(vec + (stage * 2 + 0) * TA_BC, p.lse + off, TA_BC * 4, &full_bar[stage], lead);
                bulk_load_p(vec + (stage * 2 + 1) * TA_BC, p.dsum + off, TA_BC * 4, &full_bar[stage], lead);
                // streamed query block j x the CTA's two key blocks: adjacent in the layout, so one 1 KB copy
                if (kb_load && (!CHUNK || (kb_half[0] && kb_half[1])))
                    bulk_load_p(smem + TA_OFF_KB + stage * 2 * TA_KB_BLOCK, p.keep_bits + kb_block(p, bh, j, 2 * blockIdx.x), 2 * TA_KB_BLOCK,
                                &full_bar[stage], lead);
                else if (CHUNK && kb_load) {
#pragma unroll
                    for (int half = 0; half < 2; ++half)
                        if (kb_half[half])
                            bulk_load_p(smem + TA_OFF_KB + (stage * 2 + half) * TA_KB_BLOCK, p.keep_bits + kb_block(p, bh, j, 2 * blockIdx.x + half),
                                        TA_KB_BLOCK, &full_bar[stage], lead);
                }
            }
            if (++stage == TA_NST) { stage = 0; phase ^= 1; }
        }
        return;
    }

    // ===================================================== consumers: stationary rows [wg * 64, wg * 64 + 64) of the CTA
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int et = threadIdx.x & 127;
    const int r0 = (et >> 5) * 16 + (lane >> 2);      // local rows r0, r0 + 8 of this thread (inside the warpgroup's 64)
    const int cq = (lane & 3) * 2;                    // first of the two adjacent columns of each 8-column block
    const int srow0 = row_base + wg * 64;             // first stationary index of the warpgroup
    const uint64_t stat_row0 = (uint64_t)bh * (uint64_t)T;   // row offset into the dropout index space
    const float c2 = p.alpha * TA_LOG2E;
    constexpr bool use_drop = DROP != TA_DROP_NONE, KB = DROP == TA_DROP_BITS;
    const uint32_t sbase = smem_u32(smem);
    const uint64_t kdesc = make_smem_desc_sw128(0, 16, 1024);                  // K-major tile: rows of 128 B
    const uint64_t mdesc = make_smem_desc_sw128(0, 8192, 1024);                // MN-major tile: 8-row atoms along K
    auto kmaj = [&](uint32_t addr, int k4) { return kdesc + (uint64_t)((addr >> 4) & 0x3FFF) + (uint64_t)(k4 * 2); };
    auto mnmaj = [&](uint32_t addr, int k4) { return mdesc + (uint64_t)((addr >> 4) & 0x3FFF) + (uint64_t)(k4 * 128); };
    const uint32_t st0 = sbase + TA_OFF_STAT + wg * TA_TILE_X, st1 = st0 + TA_TILE_S;
    // keep-bit word of this thread inside a 64 x 64 block (MODE 0 / 1: this thread's (query, key) pairs, see pika_b200.h)
    const int kb_word = (et >> 5) * 32 + (lane & 3) * 8 + (lane >> 2);
    uint32_t row_salt[2];                             // MODE 0 / 1: the probability rows are this thread's rows
    float lse2[2] = {0.f, 0.f}, dsum_r[2] = {0.f, 0.f};
    int c_lo[2] = {0, 0}, c_hi[2] = {0, 0};           // CHUNK: allowed streamed interval of this thread's rows
    int wg_lo = 0, wg_hi = 0;                         // CHUNK: tiles inside [wg_lo, wg_hi) are seen whole by every row of the warpgroup
    if (CHUNK) {
        wg_lo = chunk_lo<MODE>(p, srow0 + 63);
        wg_hi = chunk_hi<MODE>(p, srow0);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int srow = srow0 + r0 + 8 * hh;
        if (CHUNK) { c_lo[hh] = chunk_lo<MODE>(p, srow); c_hi[hh] = chunk_hi<MODE>(p, srow); }
        if (MODE == 0 || (MODE == 1 && !KB)) row_salt[hh] = drop_row_salt(stat_row0 + (uint64_t)srow, p.seed);
        if (MODE == 1 && srow < T) {
            lse2[hh] = p.lse[(size_t)bh * p.Tpad + srow] * TA_LOG2E;
            dsum_r[hh] = p.dsum[(size_t)bh * p.Tpad + srow];
        }
    }

    float acc0[32], acc1[32];                         // MODE 0: O | MODE 1: dQ | MODE 2: dK, dV
#pragma unroll
    for (int c = 0; c < 32; ++c) { acc0[c] = 0.f; acc1[c] = 0.f; }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    mbar_wait(stat_full, 0);
    if (MODE == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int j = j_begin; j < j_end; ++j) {
            const int col0 = j * TA_BC;
            const int nvalid = min(TA_BC, T - col0);  // streamed indices of this tile inside the sequence
            mbar_wait(&full_bar[stage], phase);
            const uint32_t x1 = sbase + TA_OFF_RING + stage * 2 * TA_TILE_X, x2 = x1 + TA_TILE_X;
            float s[32];
            wgmma_fence_acc(s);
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) wgmma_ss_n64<0, 0>(s, kmaj(st0, k4), kmaj(x1, k4), k4 > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(s);
            if (CHUNK) {
                if (col0 < wg_lo || col0 + TA_BC > wg_hi) {   // uniform; covers the keys beyond the sequence too (c_hi <= T)
#pragma unroll
                    for (int c = 0; c < 32; ++c) {
                        const int col = col0 + (c >> 2) * 8 + cq + (c & 1);
                        if (col < c_lo[(c >> 1) & 1] || col >= c_hi[(c >> 1) & 1]) s[c] = -INFINITY;
                    }
                }
            } else if (nvalid < TA_BC) {              // last tile only (uniform): keys beyond the sequence get probability 0
#pragma unroll
                for (int c = 0; c < 32; ++c) if ((c >> 2) * 8 + cq + (c & 1) >= nvalid) s[c] = -INFINITY;
            }
            uint32_t kbits = 0u;
            float corr[2];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float mx = -INFINITY;
#pragma unroll
                for (int nb = 0; nb < 8; ++nb) mx = fmaxf(mx, fmaxf(s[nb * 4 + 2 * hh], s[nb * 4 + 2 * hh + 1]));
                const float m_new = fmaxf(m_run[hh], quad_max(mx) * c2);   // finite unless CHUNK: every tile holds a valid column
                // CHUNK: a row that has seen only masked keys keeps m = -inf; its exponents use 0 instead, so that no
                // exp(-inf - (-inf)) is formed (its probabilities and corr are then exactly 0)
                const float m_use = (CHUNK && m_new == -INFINITY) ? 0.f : m_new;
                corr[hh] = ex2_approx(m_run[hh] - m_use);                    // 0 on the first tile
                float sum = 0.f;
#pragma unroll
                for (int nb = 0; nb < 8; ++nb) {
                    float* pr = &s[nb * 4 + 2 * hh];
                    pr[0] = ex2_approx(fmaf(pr[0], c2, -m_use));
                    pr[1] = ex2_approx(fmaf(pr[1], c2, -m_use));
                    sum += pr[0] + pr[1];
                    if (use_drop) {
                        const uint32_t km = drop_pair(row_salt[hh], (uint32_t)((col0 + nb * 8 + cq) >> 1), p.thresh16);
                        if (!(km & 1u)) pr[0] = 0.f;
                        if (!(km & 2u)) pr[1] = 0.f;
                        kbits |= km << (hh * 16 + nb * 2);
                    }
                }
                l_run[hh] = l_run[hh] * corr[hh] + sum;   // this thread's columns only; the quad is summed at the end
                m_run[hh] = m_new;
            }
            // streaming store: the backward reads the bits long after the rest of the step has cycled L2
            if (KB) __stcs(p.keep_bits + kb_block(p, bh, 2 * blockIdx.x + wg, j) + kb_word, kbits);
            // every A fragment is packed before the fence, so ptxas need not fence again between the register-fed wgmma
            uint32_t a[4][4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) frag_a(s, kk, a[kk]);
#pragma unroll
            for (int c = 0; c < 32; ++c) acc0[c] *= corr[(c >> 1) & 1];
            wgmma_fence_acc(acc0);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_rs_n64<1>(acc0, a[kk], mnmaj(x2, kk), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(acc0);
            if (et == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == TA_NST) { stage = 0; phase ^= 1; }
        }
    } else {
        int stage = 0;
        uint32_t phase = 0;
        for (int j = j_begin; j < j_end; ++j) {
            const int col0 = j * TA_BC;
            const bool part = CHUNK && (col0 < wg_lo || col0 + TA_BC > wg_hi);   // uniform: some pair of the tile is masked
            uint32_t kw = 0u;                             // MODE 1: keep bits of this tile, loaded under the wgmma below
            if (MODE == 1 && KB && use_drop) kw = __ldg(p.keep_bits + kb_block(p, bh, 2 * blockIdx.x + wg, j) + kb_word);
            mbar_wait(&full_bar[stage], phase);
            const uint32_t x1 = sbase + TA_OFF_RING + stage * 2 * TA_TILE_X, x2 = x1 + TA_TILE_X;
            float s[32], dp[32];
            wgmma_fence_acc(s);
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) wgmma_ss_n64<0, 0>(s, kmaj(st0, k4), kmaj(x1, k4), k4 > 0 ? 1u : 0u);
            wgmma_fence_acc(dp);
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) wgmma_ss_n64<0, 0>(dp, kmaj(st1, k4), kmaj(x2, k4), k4 > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(s);
            wgmma_fence_acc(dp);
            {
                float pd[32], ds[32];
                const float* lse_t = vec + (stage * 2 + 0) * TA_BC;
                const float* dsum_t = lse_t + TA_BC;
                // MODE 2: the probability rows of this tile are the streamed queries (this thread's columns), the keys are this thread's
                // rows.  Query q = nb*8 + cq + e, key w*16 + lane/4 + 8hh of the warpgroup's block sit in word (nb/2)*32 + (lane/8)*8 +
                // cq + e at bit (nb%2)*16 + 4w + 2hh + (lane/4)%2: four 8-byte loads give the tile's 32 bits
                uint32_t kq[4][2], qsalt[16];
                if (MODE == 2 && !KB && use_drop) {
                    // without bits: one salt per streamed query (the probability rows of this tile)
#pragma unroll
                    for (int c = 0; c < 16; ++c) qsalt[c] = drop_row_salt(stat_row0 + (uint64_t)(col0 + (c >> 1) * 8 + cq + (c & 1)), p.seed);
                }
                if (MODE == 2 && KB && use_drop) {
                    const uint32_t kb_addr = sbase + TA_OFF_KB + (stage * 2 + wg) * TA_KB_BLOCK + ((lane >> 3) * 8 + cq) * 4;
                    const int sh = (et >> 5) * 4 + ((lane >> 2) & 1);
#pragma unroll
                    for (int m = 0; m < 4; ++m) {
                        const uint2 v = lds_u32x2(kb_addr + m * 128);
                        kq[m][0] = v.x >> sh;
                        kq[m][1] = v.y >> sh;
                    }
                }
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                    for (int nb = 0; nb < 8; ++nb) {
                        uint32_t keep = 3u;
                        if (use_drop) {
                            if (MODE == 1) {
                                keep = KB ? (kw >> (hh * 16 + nb * 2)) & 3u
                                          : drop_pair(row_salt[hh], (uint32_t)((col0 + nb * 8 + cq) >> 1), p.thresh16);
                            } else if (KB) {
                                const int bit = (nb & 1) * 16 + 2 * hh;
                                keep = ((kq[nb >> 1][0] >> bit) & 1u) | (((kq[nb >> 1][1] >> bit) & 1u) << 1);
                            } else {
                                // probability row = streamed query, key = this thread's row
                                const uint32_t key = (uint32_t)(srow0 + r0 + 8 * hh);
                                const uint32_t bit = (key & 1u) ? 2u : 1u;
                                keep = ((drop_pair(qsalt[2 * nb], key >> 1, p.thresh16) & bit) ? 1u : 0u) |
                                       ((drop_pair(qsalt[2 * nb + 1], key >> 1, p.thresh16) & bit) ? 2u : 0u);
                            }
                        }
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = nb * 4 + 2 * hh + e;
                            const int cl = nb * 8 + cq + e;           // streamed index inside the tile
                            const float l2 = (MODE == 1) ? lse2[hh] : lse_t[cl] * TA_LOG2E;
                            const float dd = (MODE == 1) ? dsum_r[hh] : dsum_t[cl];
                            float pr = ex2_approx(fmaf(s[c], c2, -l2));
                            if (CHUNK && part && (col0 + cl < c_lo[hh] || col0 + cl >= c_hi[hh])) pr = 0.f;
                            const bool kp = (keep >> e) & 1u;
                            const float dpe = kp ? dp[c] * p.drop_scale : 0.f;
                            ds[c] = pr * (dpe - dd);
                            if (MODE == 2) pd[c] = kp ? pr * p.drop_scale : 0.f;
                        }
                    }
                }
                uint32_t a[4][4], a2[4][4];                   // packed before the fence, as in the forward
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    frag_a(ds, kk, a[kk]);
                    if (MODE == 2) frag_a(pd, kk, a2[kk]);
                }
                wgmma_fence_acc(acc0);
                if (MODE == 2) wgmma_fence_acc(acc1);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    wgmma_rs_n64<1>(acc0, a[kk], mnmaj(x1, kk), 1u);                    // MODE 1: dQ += dS K;  MODE 2: dK += dS^T Q
                    if (MODE == 2) wgmma_rs_n64<1>(acc1, a2[kk], mnmaj(x2, kk), 1u);    // dV += Pd^T dO
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(acc0);
            if (MODE == 2) wgmma_fence_acc(acc1);
            if (et == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == TA_NST) { stage = 0; phase ^= 1; }
        }
    }

    // ---- epilogue
    if (MODE == 0) {
        float inv[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const float l = quad_sum(l_run[hh]);
            inv[hh] = p.drop_scale / l;
            const int srow = srow0 + r0 + 8 * hh;
            // rows in [T, Tpad) (zero queries: lse = ln(T)) are written too, so that the dK/dV mode, which streams whole 64-query
            // tiles of lse, never reads a value the caller left there (a NaN would reach dK / dV through 0 * NaN)
            // CHUNK: a padding row may see no key at all (l = 0); its lse is written as 0 (the backward masks it)
            if ((lane & 3) == 0 && srow < p.Tpad) p.lse[(size_t)bh * p.Tpad + srow] = (CHUNK && l == 0.f) ? 0.f : (m_run[hh] + log2f(l)) * TA_LN2;
        }
#pragma unroll
        for (int c = 0; c < 32; ++c) acc0[c] *= inv[(c >> 1) & 1];
        store_tile(acc0, p.out + (long long)b * T * p.ld_o + h * 64, p.ld_o, srow0, T, r0, cq, 1.f);
    } else if (MODE == 1) {
        store_tile(acc0, p.dq + (long long)b * T * p.ld_dqkv + h * 64, p.ld_dqkv, srow0, T, r0, cq, p.alpha);
    } else {
        store_tile(acc0, p.dk + (long long)b * T * p.ld_dqkv + h * 64, p.ld_dqkv, srow0, T, r0, cq, p.alpha);
        store_tile(acc1, p.dv + (long long)b * T * p.ld_dqkv + h * 64, p.ld_dqkv, srow0, T, r0, cq, 1.f);
    }
}

// D[(b*heads + h)*Tpad + t] = sum_d dO[b,t,h,d] * O[b,t,h,d]; one warp per (b, t, h)
__global__ void __launch_bounds__(256) attention_rowdot_tc_kernel(const __nv_bfloat16* __restrict__ o, long long ld_o,
                                                                  const __nv_bfloat16* __restrict__ dout, long long ld_do, float* __restrict__ dsum,
                                                                  int B, int T, int heads, int Tpad) {
    const int lane = threadIdx.x & 31;
    const long long n = (long long)B * T * heads;
    for (long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); w < n; w += (long long)gridDim.x * 8) {
        const int h = (int)(w % heads);
        const long long bt = w / heads;
        const int tt = (int)(bt % T);
        const int b = (int)(bt / T);
        const uint32_t ov = *reinterpret_cast<const uint32_t*>(o + bt * ld_o + h * 64 + lane * 2);
        const uint32_t dv = *reinterpret_cast<const uint32_t*>(dout + bt * ld_do + h * 64 + lane * 2);
        const float s = warp_sum(bf16lo(ov) * bf16lo(dv) + bf16hi(ov) * bf16hi(dv));
        if (lane == 0) dsum[((long long)b * heads + h) * Tpad + tt] = s;
    }
    // D of the padding rows [T, Tpad) is 0, for the same reason as the forward's lse padding
    const long long npad = (long long)B * heads * (Tpad - T);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npad; i += (long long)gridDim.x * blockDim.x)
        dsum[(i / (Tpad - T)) * Tpad + T + i % (Tpad - T)] = 0.f;
}

static int attn_maps(AttnTcParams& p, const void* q, const void* k, const void* v, long long ld_qkv, const void* dout, long long ld_dout) {
    const unsigned long long dims[3] = {(unsigned long long)p.heads * 64, (unsigned long long)p.T, (unsigned long long)p.B};
    const unsigned box[3] = {64, TA_BC, 1};
    const unsigned long long st_qkv[2] = {(unsigned long long)ld_qkv * 2, (unsigned long long)ld_qkv * 2 * p.T};
    int rc;
    if ((rc = encode_tiled_bf16_3d(&p.q, q, dims, st_qkv, box, "attention q"))) return rc;
    if ((rc = encode_tiled_bf16_3d(&p.k, k, dims, st_qkv, box, "attention k"))) return rc;
    if ((rc = encode_tiled_bf16_3d(&p.v, v, dims, st_qkv, box, "attention v"))) return rc;
    if (dout) {
        const unsigned long long st_do[2] = {(unsigned long long)ld_dout * 2, (unsigned long long)ld_dout * 2 * p.T};
        if ((rc = encode_tiled_bf16_3d(&p.dout, dout, dims, st_do, box, "attention dout"))) return rc;
    }
    return 0;
}

template <int MODE, int DROP, bool CHUNK> static int launch_attn_drop(const AttnTcParams& p, cudaStream_t st) {
    auto kern = attention_tc_kernel<MODE, DROP, CHUNK>;
    static bool configured = false;
    if (!configured) {
        PK_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TA_SMEM));
        configured = true;
    }
    dim3 grid((p.T + TA_BR - 1) / TA_BR, p.B * p.heads);
    kern<<<grid, TA_THREADS, TA_SMEM, st>>>(p);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
template <int MODE> static int launch_attn(const AttnTcParams& p, cudaStream_t st) {
    if (p.chunk_len > 0) {                        // chunk mask: keep-bits form only
        if (p.thresh16 == 0u) return launch_attn_drop<MODE, TA_DROP_NONE, true>(p, st);
        return launch_attn_drop<MODE, TA_DROP_BITS, true>(p, st);
    }
    if (p.thresh16 == 0u) return launch_attn_drop<MODE, TA_DROP_NONE, false>(p, st);
    return p.keep_bits ? launch_attn_drop<MODE, TA_DROP_BITS, false>(p, st) : launch_attn_drop<MODE, TA_DROP_HASH, false>(p, st);
}

}  // namespace pk

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int pk_attention_lse_stride(int T) { return (T + 63) / 64 * 64; }
static int attn_kb_blocks(int T) { return (T + 127) / 128 * 2; }
extern "C" long long pk_attention_keep_bits_bytes(int B, int T, int heads) {
    const long long n = attn_kb_blocks(T);
    return (long long)B * heads * n * n * pk::TA_KB_BLOCK;
}

#define ATTN_CHECKS()                                                                                                      \
    PK_CHECK_ARG(B > 0 && T > 0 && heads > 0, "bad dims");                                                                 \
    PK_CHECK_ARG(dh == 64, "fused attention supports head dim 64");                                                        \
    PK_CHECK_ARG(ld_qkv % 8 == 0 && ld_out % 8 == 0, "row strides must be multiples of 8 elements (16 bytes)");            \
    PK_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f, "drop_p out of range");                                                    \
    PK_CHECK_ARG((long long)B * heads < 65536, "B * heads must be < 65536")
#define KEEP_BITS_CHECK()                                                                                                  \
    PK_CHECK_ARG(drop_p == 0.f || (keep_bits != nullptr && ((uintptr_t)keep_bits & 15) == 0),                               \
                 "keep_bits must be a 16-byte aligned buffer of pk_attention_keep_bits_bytes when drop_p > 0")

#define CHUNK_CHECKS()                                                                                                     \
    PK_CHECK_ARG(chunk_len >= 1 && chunk_off >= 0 && left_chunks >= -1, "chunk mask: chunk_len >= 1, chunk_off >= 0, left_chunks >= -1")

/* 1 when the chunk mask (chunk_len, chunk_off, left_chunks) lets every query of a T-frame sequence see every key: the last query's
   lowest key is 0 and the first query's highest key is T - 1 (both ends are monotone in the query) */
extern "C" int pk_attention_chunk_admits_all(int T, int chunk_len, int chunk_off, int left_chunks) {
    CHUNK_CHECKS();
    PK_CHECK_ARG(T > 0, "bad dims");
    return pk::chunk_key_lo(T - 1, T, chunk_len, chunk_off, left_chunks) == 0 && pk::chunk_key_hi(0, T, chunk_len, chunk_off) == T;
}

static int attention_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                         int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, uint32_t* keep_bits, void* stream,
                         int chunk_len = 0, int chunk_off = 0, int left_chunks = -1) {
    using namespace pk;
    ATTN_CHECKS();
    static thread_local AttnTcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.T = T; p.heads = heads; p.Tpad = pk_attention_lse_stride(T); p.Tp2 = (T + 1) / 2;
    p.keep_bits = drop_p > 0.f ? keep_bits : nullptr; p.nkb = attn_kb_blocks(T);
    int rc = attn_maps(p, q, k, v, ld_qkv, nullptr, 0);
    if (rc) return rc;
    p.out = (__nv_bfloat16*)out; p.ld_o = ld_out; p.lse = lse;
    p.chunk_len = chunk_len; p.chunk_off = chunk_off; p.left_chunks = left_chunks;
    p.alpha = alpha;
    p.thresh16 = drop_thresh16_of(drop_p); p.drop_scale = drop_scale16_of(p.thresh16); p.seed = seed;
    return launch_attn<0>(p, STREAM(stream));
}

/* dq/dk/dv share the row stride ld_dqkv (the fused [B,T,3D] gradient buffer); lse and dsum_ws: [B*heads][pk_attention_lse_stride(T)],
   whose padding t in [T, stride) the kernels write themselves (lse in the forward, dsum_ws here): neither needs initialising.
   keep_bits NULL: the kernels hash the mask from seed */
static int attention_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                         const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                         long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed,
                         const uint32_t* keep_bits, void* stream, int chunk_len = 0, int chunk_off = 0, int left_chunks = -1) {
    using namespace pk;
    ATTN_CHECKS();
    PK_CHECK_ARG(ld_dout % 8 == 0 && ld_dqkv % 8 == 0, "row strides must be multiples of 8 elements (16 bytes)");
    static thread_local AttnTcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.T = T; p.heads = heads; p.Tpad = pk_attention_lse_stride(T); p.Tp2 = (T + 1) / 2;
    p.keep_bits = drop_p > 0.f ? const_cast<uint32_t*>(keep_bits) : nullptr; p.nkb = attn_kb_blocks(T);
    int rc = attn_maps(p, q, k, v, ld_qkv, dout, ld_dout);
    if (rc) return rc;
    p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv; p.ld_dqkv = ld_dqkv;
    p.lse = const_cast<float*>(lse); p.dsum = dsum_ws;
    p.chunk_len = chunk_len; p.chunk_off = chunk_off; p.left_chunks = left_chunks;
    p.alpha = alpha;
    p.thresh16 = drop_thresh16_of(drop_p); p.drop_scale = drop_scale16_of(p.thresh16); p.seed = seed;
    const long long n = (long long)B * T * heads;
    const long long rmax = (long long)num_sms() * 16;
    const int rgrid = (int)((n + 7) / 8 < rmax ? (n + 7) / 8 : rmax);
    attention_rowdot_tc_kernel<<<rgrid, 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)out, ld_out, (const __nv_bfloat16*)dout, ld_dout, dsum_ws,
                                                                   B, T, heads, p.Tpad);
    PK_CHECK_LAUNCH(); count_launch();
    rc = launch_attn<1>(p, STREAM(stream));
    if (rc) return rc;
    return launch_attn<2>(p, STREAM(stream));
}

extern "C" int pk_attention_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                                int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, void* stream) {
    return attention_fwd(q, k, v, ld_qkv, out, ld_out, lse, B, T, heads, dh, alpha, drop_p, seed, nullptr, stream);
}
extern "C" int pk_attention_fwd_bits(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                                     int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, uint32_t* keep_bits,
                                     void* stream) {
    KEEP_BITS_CHECK();
    return attention_fwd(q, k, v, ld_qkv, out, ld_out, lse, B, T, heads, dh, alpha, drop_p, seed, keep_bits, stream);
}
extern "C" int pk_attention_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                                const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                                long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, void* stream) {
    return attention_bwd(q, k, v, ld_qkv, out, ld_out, dout, ld_dout, lse, dsum_ws, dq, dk, dv, ld_dqkv, B, T, heads, dh, alpha, drop_p, seed,
                         nullptr, stream);
}
extern "C" int pk_attention_bwd_bits(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                                     const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                                     long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, const uint32_t* keep_bits,
                                     void* stream) {
    KEEP_BITS_CHECK();
    return attention_bwd(q, k, v, ld_qkv, out, ld_out, dout, ld_dout, lse, dsum_ws, dq, dk, dv, ld_dqkv, B, T, heads, dh, alpha, drop_p, 0u,
                         keep_bits, stream);
}

/* chunk-masked forms; a mask that admits every key runs the unmasked kernels */
extern "C" int pk_attention_fwd_chunk(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                                      int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, uint32_t* keep_bits,
                                      int chunk_len, int chunk_off, int left_chunks, void* stream) {
    CHUNK_CHECKS();
    KEEP_BITS_CHECK();
    ATTN_CHECKS();
    if (pk_attention_chunk_admits_all(T, chunk_len, chunk_off, left_chunks)) chunk_len = 0;
    return attention_fwd(q, k, v, ld_qkv, out, ld_out, lse, B, T, heads, dh, alpha, drop_p, seed, keep_bits, stream, chunk_len, chunk_off,
                         left_chunks);
}
extern "C" int pk_attention_bwd_chunk(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                                      const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                                      long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, const uint32_t* keep_bits,
                                      int chunk_len, int chunk_off, int left_chunks, void* stream) {
    CHUNK_CHECKS();
    KEEP_BITS_CHECK();
    ATTN_CHECKS();
    if (pk_attention_chunk_admits_all(T, chunk_len, chunk_off, left_chunks)) chunk_len = 0;
    return attention_bwd(q, k, v, ld_qkv, out, ld_out, dout, ld_dout, lse, dsum_ws, dq, dk, dv, ld_dqkv, B, T, heads, dh, alpha, drop_p, 0u,
                         keep_bits, stream, chunk_len, chunk_off, left_chunks);
}
