// wgmma / TMA GEMM for sm_90a: C = epilogue(alpha * sum_p A_p * B_p^T).
//
// One persistent CTA per SM, three warpgroups per CTA:
//   warp 0           TMA producer   (one converged warp: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx)
//   warps 1-3        epilogue       (bf16 C with the plain or LSE epilogue: TMA-store the finished C tile from shared memory, hand it
//                                    back; stage the next tile's bias)
//   warpgroups 1, 2  consumers      (wgmma m64 x BN x k16 from shared-memory descriptors, fp32 accumulators in registers; each
//                                    owns 64 rows of the 128-row tile, releases ring stages one k-block behind.  bf16 plain / LSE:
//                                    alpha, bias, ReLU, bf16 rounding into the C tile with stmatrix, then straight on to the next
//                                    tile's main loop.  LSE: the row max comes from the registers being rounded; the exp-sum reads the
//                                    warp's own rows of the C tile back while the next tile's wgmma run.  EPI_FULL and f32 C: the whole
//                                    epilogue, registers -> swizzled smem -> TMA store / TMA reduce-add, in 64-column chunks)
// Tile 128 x BN x 64 per CTA (BN = 64 | 128 | 256).  Operands may be K-major or MN-major (wgrad / dgrad / P.V use the MN-major form so no
// transposes are ever materialised).  Up to 9 (A,B) pairs accumulate into one tile (TDNN taps, split-bf16 fp32-class mode), plus a
// batched reduction loop (kz) for per-utterance wgrad, plus split-K.
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KB
constexpr int C_STAGE_BYTES = 64 * 128;      // one consumer's 64 rows x 128 B
constexpr int CONSUMERS = 2;

struct GemmParams {
    CUtensorMap a[PK_GEMM_MAX_PAIRS];
    CUtensorMap b[PK_GEMM_MAX_PAIRS];
    CUtensorMap c;
    int a_off[PK_GEMM_MAX_PAIRS];
    int b_off[PK_GEMM_MAX_PAIRS];
    int n_pairs, kz_count, num_k_blocks;
    int k_splits, iters_per_split;      // split-K over the flattened (pair, kz, k-block) iteration space
    int M, N, tiles_m, tiles_n, zb0, zb1;   // tiles_m / tiles_n: BM-row / BN-column tiles of one C matrix
    int a_sel2, a_sel3, b_sel2, b_sel3;
    int c_is_f32, c_accumulate;
    float alpha;
    const float* bias;
    int act;
    uint32_t drop_thresh;
    float drop_scale;
    uint32_t drop_seed;
    int aux_mode, aux_is_f32;
    const void* aux;
    long long aux_sm, aux_s0, aux_s1;
    float aux_scale;
    float* row_lse;                     // optional [tiles_n][M][2] per-row (max*log2e, sum 2^(x*log2e-max)) partials of the bf16 output
    uint64_t pol_a, pol_b, pol_c;       // L2 eviction priorities of the three streams
    const int* a_rows_dev;              // optional: rows of A counted on the device (pk_gemm_desc.a_rows_dev)
};

// EPI_WARPS: warps 1-3 TMA-store a whole BM x BN bf16 C tile from shared memory (bf16 C, EPI_PLAIN / EPI_LSE).
// Otherwise the consumers stage 64-column chunks through two small buffers each.  The C tile costs BN = 256 its fourth ring stage.
template <int BN, bool EPI_WARPS> struct GemmCfg {
    static constexpr int B_STAGE_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    static constexpr int STAGES = BN == 256 ? (EPI_WARPS ? 3 : 4) : (BN == 128 ? 6 : 8);
    static constexpr int C_OFF = STAGES * STAGE_BYTES;
    static constexpr int C_BYTES = EPI_WARPS ? BM * BN * 2 : CONSUMERS * 2 * C_STAGE_BYTES;
    static constexpr int BIAS_OFF = C_OFF + C_BYTES;                    // EPI_WARPS: the tile's BN bias values (f32)
    static constexpr int BAR_OFF = BIAS_OFF + (EPI_WARPS ? BN * 4 : 0);
    static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024;             // + barriers + alignment slack
    static constexpr int THREADS = 128 + CONSUMERS * 128;
    static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

PK_DEVICE int pick_sel(int sel, int zb0, int zb1, int kz) {
    return sel == PK_SEL_ZB0 ? zb0 : (sel == PK_SEL_ZB1 ? zb1 : (sel == PK_SEL_KZ ? kz : 0));
}

struct UnitCoord { int mb, nb, zb0, zb1, split; };
// work unit -> (output tile, K split).  Units run split-major: all tiles of split 0, then split 1, ..., so CTAs that run together
// share a k-window.
PK_DEVICE UnitCoord decode_unit(const GemmParams& p, int unit) {
    UnitCoord u;
    const int tiles_per_z = p.tiles_m * p.tiles_n;
    const int out_tiles = tiles_per_z * p.zb0 * p.zb1;
    u.split = unit / out_tiles;
    const int tile = unit - u.split * out_tiles;
    const int z = tile / tiles_per_z;
    const int r = tile - z * tiles_per_z;
    u.mb = r / p.tiles_n; u.nb = r - u.mb * p.tiles_n;
    u.zb1 = z / p.zb0; u.zb0 = z - u.zb1 * p.zb0;
    return u;
}

template <int BN, bool A_MN, bool B_MN> PK_DEVICE void wgmma_tile(float (&acc)[BN / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
    if constexpr (BN == 64) wgmma_ss_n64<A_MN, B_MN>(acc, a, b, accumulate);
    else if constexpr (BN == 128) wgmma_ss_n128<A_MN, B_MN>(acc, a, b, accumulate);
    else wgmma_ss_n256<A_MN, B_MN>(acc, a, b, accumulate);
}

// EPI selects what the epilogue compiles in, so that the common case is straight-line code:
//   EPI_PLAIN  alpha, bias, ReLU only      EPI_LSE  + per-row log-sum-exp partials (bf16 C)      EPI_FULL  + dropout / aux add / aux mask
enum { EPI_PLAIN = 0, EPI_LSE = 1, EPI_FULL = 2 };
// EPI_FULL and f32 C (wgrad, split-K reduce-add) keep the epilogue in the consumers: their K is long or they are off the joint's path,
// so the tensor-pipe idle time it causes is small.
template <bool CF32, int EPI> constexpr bool epi_warps() { return !CF32 && EPI != EPI_FULL; }

template <bool A_MN, bool B_MN, int BN, bool CF32, int EPI>
__global__ void __launch_bounds__(GemmCfg<BN, epi_warps<CF32, EPI>()>::THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ GemmParams p) {
    constexpr bool EW = epi_warps<CF32, EPI>();
    static_assert(EPI != EPI_LSE || (EW && BN == 256), "the row log-sum-exp epilogue works on bf16 256-wide tiles");
    using Cfg = GemmCfg<BN, EW>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
    uint64_t* empty_bar = full_bar + Cfg::STAGES;
    // EW: the C tile is full (8 consumer warps have written it) / empty (its TMA store has read it, the epilogue warps have staged the next bias)
    uint64_t* c_full = empty_bar + Cfg::STAGES;
    uint64_t* c_empty = c_full + 1;
    const uint32_t ctile = smem_u32(smem + Cfg::C_OFF);                 // EW: [BN / 64][BM rows][128 B], TMA 128B swizzle
    const uint32_t sbias = smem_u32(smem + Cfg::BIAS_OFF);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int worker = (int)blockIdx.x, n_workers = (int)gridDim.x;    // persistent CTAs stride over the work units

    if (threadIdx.x == 0) {
        for (int i = 0; i < p.n_pairs; ++i) {
            tma_prefetch_desc(&p.a[i]);
            tma_prefetch_desc(&p.b[i]);
        }
        tma_prefetch_desc(&p.c);
        for (int s = 0; s < Cfg::STAGES; ++s) {
            mbar_init(&full_bar[s], 1);              // the producer's expect_tx arrive
            mbar_init(&empty_bar[s], CONSUMERS);     // one arrive per consumer warpgroup
        }
        if (EW) {
            mbar_init(c_full, CONSUMERS * 4);
            mbar_init(c_empty, 3);
        }
        mbar_fence_init();
    }
    __syncthreads();

    const int out_tiles = p.tiles_m * p.tiles_n * p.zb0 * p.zb1;
    int num_units = out_tiles * p.k_splits;                             // work units = tiles x K-splits
    int k_iters_total = p.n_pairs * p.kz_count * p.num_k_blocks;
    int ips = p.iters_per_split;
    if (p.a_rows_dev != nullptr) {
        // the host allows this with one pair, kz_count 1 and a 2-D C, so units run m-tile-major and the k-blocks are K / BK
        const int rows = *p.a_rows_dev;
        if (A_MN) {                                                     // rows are K: shorten the reduction, re-cut it into the splits
            k_iters_total = min(k_iters_total, (rows + BK - 1) / BK);
            ips = max(1, (k_iters_total + p.k_splits - 1) / p.k_splits);
        } else {                                                        // rows are M: drop the tiles past the last row
            num_units = min(num_units, (rows + BM - 1) / BM * p.tiles_n);
        }
    }

    if (warp < 4) {
        setmaxnreg_dec<40>();
    }
    if (warp == 0) {
        // ===================================================== TMA producer (converged warp; one elected lane issues, common.cuh)
        const uint32_t lead = elect_one_u32();
        int stage = 0;
        uint32_t phase = 0;
        const int kzb = p.kz_count * p.num_k_blocks;
        for (int unit = worker; unit < num_units; unit += n_workers) {
            const UnitCoord u = decode_unit(p, unit);
            const int m0 = u.mb * BM, n0 = u.nb * BN;
            const int i0 = u.split * ips, i1 = min(k_iters_total, i0 + ips);
            // position in the flattened (pair, kz, k-block) space: decoded once per unit, then advanced by counters
            int pr = i0 / kzb;
            int rem = i0 - pr * kzb;
            int kz = rem / p.num_k_blocks, kb = rem - kz * p.num_k_blocks;
            int a2 = pick_sel(p.a_sel2, u.zb0, u.zb1, kz), a3 = pick_sel(p.a_sel3, u.zb0, u.zb1, kz);
            int b2 = pick_sel(p.b_sel2, u.zb0, u.zb1, kz), b3 = pick_sel(p.b_sel3, u.zb0, u.zb1, kz);
            const CUtensorMap* ma = &p.a[pr];
            const CUtensorMap* mbp = &p.b[pr];
            int a_off = p.a_off[pr], b_off = p.b_off[pr];
            for (int i = i0; i < i1; ++i) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                uint8_t* sb = sa + A_STAGE_BYTES;
                mbar_arrive_expect_tx_p(&full_bar[stage], Cfg::STAGE_BYTES, lead);
                const int k0 = kb * BK;
                if (A_MN) {
#pragma unroll
                    for (int c = 0; c < BM / 64; ++c)
                        tma_load_4d_hint_p(sa + c * (64 * BK * 2), ma, &full_bar[stage], m0 + c * 64, k0 + a_off, a2, a3, p.pol_a, lead);
                } else {
                    tma_load_4d_hint_p(sa, ma, &full_bar[stage], k0, m0 + a_off, a2, a3, p.pol_a, lead);
                }
                if (B_MN) {
#pragma unroll
                    for (int c = 0; c < BN / 64; ++c)
                        tma_load_4d_hint_p(sb + c * (64 * BK * 2), mbp, &full_bar[stage], n0 + c * 64, k0 + b_off, b2, b3, p.pol_b, lead);
                } else {
                    tma_load_4d_hint_p(sb, mbp, &full_bar[stage], k0, n0 + b_off, b2, b3, p.pol_b, lead);
                }
                if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
                if (++kb == p.num_k_blocks) {
                    kb = 0;
                    if (++kz == p.kz_count) {
                        kz = 0;
                        if (++pr < p.n_pairs) { ma = &p.a[pr]; mbp = &p.b[pr]; a_off = p.a_off[pr]; b_off = p.b_off[pr]; }
                    }
                    a2 = pick_sel(p.a_sel2, u.zb0, u.zb1, kz); a3 = pick_sel(p.a_sel3, u.zb0, u.zb1, kz);
                    b2 = pick_sel(p.b_sel2, u.zb0, u.zb1, kz); b3 = pick_sel(p.b_sel3, u.zb0, u.zb1, kz);
                }
            }
        }
    }
    if (EW && warp >= 1 && warp < 4) {
        // ===================================================== epilogue warps: bias staging, TMA stores of the C tile
        const int et = threadIdx.x - 32;
        const uint32_t store_pred = (threadIdx.x == 32) ? 1u : 0u;
        uint32_t cph = 0;
        for (int unit = worker; unit < num_units; unit += n_workers, cph ^= 1) {
            const UnitCoord u = decode_unit(p, unit);
            const int m0 = u.mb * BM, n0 = u.nb * BN;
            // the consumers read the previous tile's bias before they marked C full, which this warp waited for
            for (int c = et; c < BN; c += 96) sts_f32(sbias + c * 4, (p.bias != nullptr && n0 + c < p.N) ? __ldg(p.bias + n0 + c) : 0.f);
            __syncwarp();
            if (lane == 0) mbar_arrive(c_empty);
            mbar_wait(c_full, cph);
#pragma unroll
            for (int ch = 0; ch < BN / 64; ++ch)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (n0 + ch * 64 < p.N && m0 + h * 64 < p.M)
                        tma_store_4d_hint_p(&p.c, smem + Cfg::C_OFF + ch * (BM * 128) + h * (64 * 128), n0 + ch * 64, m0 + h * 64, u.zb0, u.zb1,
                                            p.pol_c, store_pred);
            tma_store_commit_p(store_pred);
            tma_store_wait_read_p<0>(store_pred);      // the TMA has read the tile: the consumers may overwrite it
        }
        if (store_pred) tma_store_wait<0>();
    }
    if (warp >= 4) {
    // ===================================================== consumers: MMA + epilogue for rows [wg * 64, wg * 64 + 64) of each tile
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int et = threadIdx.x & 127;                  // thread inside the warpgroup
    const int w4 = et >> 5;                            // warp inside the warpgroup
    const uint32_t store_pred = (et == 0) ? 1u : 0u;   // the warpgroup's first thread owns the TMA stores
    const int bar_stage = 1 + wg;
    constexpr int GW = CF32 ? 4 : 8;                   // columns per 16-byte group
    constexpr int CH = 8 * GW;                         // columns per 128-byte staging row
    constexpr int ES = CF32 ? 4 : 2;
    uint8_t* cst = smem + Cfg::C_OFF + wg * 2 * C_STAGE_BYTES;
    const float relu_floor = (p.act == PK_ACT_RELU) ? 0.f : -INFINITY;
    // A: this warpgroup's 64 rows start 8192 B into the stage for both layouts (64 K-major rows of 128 B, or the second 64-wide MN chunk)
    const uint32_t base16 = (smem_u32(smem) >> 4) & 0x3FFF;
    const uint64_t a_desc0 = (A_MN ? make_smem_desc_sw128(0, 64 * BK * 2, 1024) : make_smem_desc_sw128(0, 16, 1024)) + base16 + ((wg * 8192) >> 4);
    const uint64_t b_desc0 = (B_MN ? make_smem_desc_sw128(0, 64 * BK * 2, 1024) : make_smem_desc_sw128(0, 16, 1024)) + base16 + (A_STAGE_BYTES >> 4);
    constexpr uint32_t A_K16 = (A_MN ? 2048 : 32) >> 4, B_K16 = (B_MN ? 2048 : 32) >> 4;
    const int r0 = w4 * 16 + (lane >> 2);              // local rows r0 and r0 + 8 of this thread
    const int cq = (lane & 3) * 2;                     // first of the two adjacent columns of each 8-column block

    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t chunk_ctr = 0;
    uint32_t cph = 0;                                  // EW: parity of the C tile's barriers
    auto release = [&](int s) {
        if (et == 0) mbar_arrive(&empty_bar[s]);
    };
    // EPI_LSE: (max * log2e, sum 2^(x * log2e - max)) of each row's rounded values.  The max is taken in registers while the tile is
    // rounded; the sum of the tile the warp wrote last is read back from its own 16 rows of the C tile in LSE_SLICES slices, one
    // per k-block of the next tile while its wgmma run (the rest after that main loop; a worker's last tile after its unit loop).
    // Those reads come before the warp's stmatrix of the next tile in program order, and the TMA store only reads: no barrier
    // beyond a __syncwarp is needed before the C tile is overwritten.  Lane quad lane / 4 owns rows r0 and r0 + 8 as in the
    // accumulators; slice t is one 16-byte chunk of row r0 + 8 * (t >> 3), 64-column block (t >> 1) & 3, chunk 2 * (lane & 3) +
    // (t & 1): each quarter warp reads all eight chunk positions of the swizzled rows, so the 16-byte loads are conflict-free.
    constexpr float L2E = 1.4426950408889634f;
    constexpr int LSE_SLICES = BN / 16;                // 16 rows x BN columns of bf16 over 32 lanes, 16 B each
    bool lse_pending = false;                          // the previous tile's sums are still to be taken
    float lse_m0 = 0.f, lse_m1 = 0.f, lse_s0 = 0.f, lse_s1 = 0.f;
    int lse_row = 0, lse_nb = 0, lse_nvalid = 0;       // global row of r0, N tile, valid columns of the pending tile
    const uint32_t lse_addr = ctile + (uint32_t)(wg * 64 + r0) * 128;
    auto lse_slice = [&](int t) {
        const int j = (t >> 1) & 3, g = (lane & 3) * 2 + (t & 1);
        if (j * 64 + g * 8 < lse_nvalid) {             // N % 8 == 0: a 16-byte chunk is valid as a whole
            const bool hi = (t >> 3) != 0;
            const uint4 v = lds_u32x4(lse_addr + (hi ? 8 * 128 : 0) + j * (BM * 128) + ((g ^ (lane >> 2)) << 4));
            const float nm = hi ? -lse_m1 : -lse_m0;
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            float s = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) s += ex2_approx(fmaf(bf16lo(w[q]), L2E, nm)) + ex2_approx(fmaf(bf16hi(w[q]), L2E, nm));
            if (hi) lse_s1 += s; else lse_s0 += s;
        }
    };
    auto lse_finish = [&]() {
        lse_s0 += __shfl_xor_sync(0xffffffffu, lse_s0, 1);
        lse_s1 += __shfl_xor_sync(0xffffffffu, lse_s1, 1);
        lse_s0 += __shfl_xor_sync(0xffffffffu, lse_s0, 2);
        lse_s1 += __shfl_xor_sync(0xffffffffu, lse_s1, 2);
        // a tile with no column below N is an empty partial (max = -inf, sum = 0), which the merges ignore
        float* dst = p.row_lse + ((size_t)lse_nb * (size_t)p.M + (size_t)lse_row) * 2;
        if ((lane & 3) == 0 && lse_row < p.M) *reinterpret_cast<float2*>(dst) = make_float2(lse_m0, lse_m0 == -INFINITY ? 0.f : lse_s0);
        if ((lane & 3) == 0 && lse_row + 8 < p.M)
            *reinterpret_cast<float2*>(dst + 16) = make_float2(lse_m1, lse_m1 == -INFINITY ? 0.f : lse_s1);
        lse_pending = false;
    };
    for (int unit = worker; unit < num_units; unit += n_workers) {
        const UnitCoord u = decode_unit(p, unit);
        const int k_iters = max(0, min(k_iters_total, (u.split + 1) * ips) - u.split * ips);
        if (k_iters == 0) {                            // a split past a device-side row count: its share of C is zero
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        }
        int prev = -1;
        for (int k = 0; k < k_iters; ++k) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t st16 = (uint32_t)(stage * Cfg::STAGE_BYTES) >> 4;
            wgmma_fence_acc(acc);
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < BK / 16; ++k4)
                wgmma_tile<BN, A_MN, B_MN>(acc, a_desc0 + st16 + k4 * A_K16, b_desc0 + st16 + k4 * B_K16, (k > 0 || k4 > 0) ? 1u : 0u);
            wgmma_commit();
            wgmma_fence_acc(acc);
            wgmma_wait<1>();                           // the previous k-block's products are done: its stage may be refilled
            if (prev >= 0) release(prev);
            // after the release, not before the wait: with a 3-stage ring, a stage handed back late stalls its refill
            if constexpr (EPI == EPI_LSE) {
                if (lse_pending && k < LSE_SLICES) lse_slice(k);
            }
            prev = stage;
            if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if (prev >= 0) release(prev);

        if constexpr (EW) {
            if constexpr (EPI == EPI_LSE) {
                if (lse_pending) {
                    for (int t = k_iters; t < LSE_SLICES; ++t) lse_slice(t);
                    lse_finish();
                }
            }
            // ------------------------------------------ alpha, bias, ReLU, RN to bf16 into the C tile; the epilogue warps take it from there
            mbar_wait(c_empty, cph);
            // LSE: every lane's reads of the previous tile come before any lane's stmatrix below.  Nothing else orders them: c_empty
            // only says that the TMA store has read the tile.
            if constexpr (EPI == EPI_LSE) __syncwarp();
            const int nvalid = p.N - u.nb * BN;
            uint32_t mx[2] = {0xFF80FF80u, 0xFF80FF80u};  // LSE: bf16 -inf pairs, the running max of rows r0 and r0 + 8
            // stmatrix.x4 per pair of 8-column blocks (2q, 2q + 1): matrices (rows r0 | r0 + 8) x (block 2q | 2q + 1); lane -> row address
            const int mi = lane >> 3;
            const uint32_t row_addr = ctile + (uint32_t)(wg * 64 + w4 * 16 + (lane & 7) + ((mi & 1) << 3)) * 128;
#pragma unroll
            for (int q = 0; q < BN / 16; ++q) {
                uint32_t r[4];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int blk = 2 * q + i;
                    const float2 bs = lds_f32x2(sbias + (blk * 8 + cq) * 4);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        r[2 * i + h] = pack_bf16x2(fmaxf(fmaf(acc[blk * 4 + 2 * h], p.alpha, bs.x), relu_floor),
                                                   fmaxf(fmaf(acc[blk * 4 + 2 * h + 1], p.alpha, bs.y), relu_floor));
                    // columns >= N hold zeros from the zero-filled B rows, not logits
                    if (EPI == EPI_LSE && blk * 8 < nvalid) { mx[0] = bf16x2_max(mx[0], r[2 * i]); mx[1] = bf16x2_max(mx[1], r[2 * i + 1]); }
                }
                const int blk = 2 * q + (mi >> 1);
                stmatrix_x4(row_addr + (blk >> 3) * (BM * 128) + (((blk & 7) ^ (lane & 7)) << 4), r[0], r[1], r[2], r[3]);
            }
            fence_proxy_async_smem();                  // the TMA store reads these bytes through the async proxy
            __syncwarp();                              // LSE: and so does this warp's exp-sum, from other lanes' stmatrix
            if (lane == 0) mbar_arrive(c_full);
            cph ^= 1;
            if constexpr (EPI == EPI_LSE) {
                // max is exact and x * log2e is monotonic: the same m as a max over the rounded tile in shared memory
                float x0 = fmaxf(bf16lo(mx[0]), bf16hi(mx[0])), x1 = fmaxf(bf16lo(mx[1]), bf16hi(mx[1]));
                x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1));
                x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1));
                x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
                x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
                lse_m0 = x0 * L2E; lse_m1 = x1 * L2E;
                lse_s0 = 0.f; lse_s1 = 0.f;
                lse_row = u.mb * BM + wg * 64 + r0;
                lse_nb = u.nb;
                lse_nvalid = nvalid;
                lse_pending = true;
            }
            continue;
        }

        // ---------------------------------------------- epilogue (EPI_FULL, f32 C)
        const int zb0 = u.zb0, zb1 = u.zb1;
        const int m0 = u.mb * BM + wg * 64;
        const int n0 = u.nb * BN;
        if (m0 >= p.M) continue;                       // uniform across the warpgroup
        const int mrow[2] = {m0 + r0, m0 + r0 + 8};
        const unsigned char* aux_row[2] = {nullptr, nullptr};
        uint64_t lin_row[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (EPI == EPI_FULL && p.aux_mode != PK_AUX_NONE && mrow[h] < p.M) {
                const long long off = (long long)mrow[h] * p.aux_sm + (long long)zb0 * p.aux_s0 + (long long)zb1 * p.aux_s1;
                aux_row[h] = reinterpret_cast<const unsigned char*>(p.aux) + off * (p.aux_is_f32 ? 4 : 2);
            }
            lin_row[h] = ((uint64_t)(zb1 * p.zb0 + zb0) * (uint64_t)p.M + (uint64_t)mrow[h]) * (uint64_t)p.N;
        }
        constexpr int n_chunks = BN / CH;
#pragma unroll
        for (int ch = 0; ch < n_chunks; ++ch) {
            const int nc0 = n0 + ch * CH;
            if (nc0 >= p.N) break;                     // uniform across the warpgroup
            uint8_t* sbuf = cst + (chunk_ctr & 1) * C_STAGE_BYTES;
            tma_store_wait_read_p<1>(store_pred);      // the buffer used two chunks ago is free
            named_bar_sync(bar_stage, 128);
#pragma unroll
            for (int nb = 0; nb < CH / 8; ++nb) {
                const int cl = nb * 8 + cq;            // column inside the chunk
                const int ncol = nc0 + cl;
                float bs[2];
                if (p.bias != nullptr && ncol < p.N) { bs[0] = __ldg(p.bias + ncol); bs[1] = (ncol + 1 < p.N) ? __ldg(p.bias + ncol + 1) : 0.f; }
                else { bs[0] = 0.f; bs[1] = 0.f; }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ai = (ch * (CH / 8) + nb) * 4 + 2 * h;
                    float x[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) x[e] = fmaxf(fmaf(acc[ai + e], p.alpha, bs[e]), relu_floor);
                    if (EPI == EPI_FULL && p.drop_thresh != 0u) {
#pragma unroll
                        for (int e = 0; e < 2; ++e)
                            x[e] = drop_keep(lin_row[h] + (uint64_t)(ncol + e), p.drop_seed, p.drop_thresh) ? x[e] * p.drop_scale : 0.f;
                    }
                    if (EPI == EPI_FULL && aux_row[h] != nullptr && ncol < p.N) {     // N % 8 == 0 is enforced on the host when aux is used
                        float a[2];
                        if (p.aux_is_f32) {
                            const float2 t2 = *reinterpret_cast<const float2*>(aux_row[h] + (size_t)ncol * 4);
                            a[0] = t2.x; a[1] = t2.y;
                        } else {
                            const uint32_t t1 = *reinterpret_cast<const uint32_t*>(aux_row[h] + (size_t)ncol * 2);
                            a[0] = bf16lo(t1); a[1] = bf16hi(t1);
                        }
                        if (p.aux_mode == PK_AUX_ADD) { x[0] += a[0]; x[1] += a[1]; }
                        else { x[0] = (a[0] != 0.f) ? x[0] * p.aux_scale : 0.f; x[1] = (a[1] != 0.f) ? x[1] * p.aux_scale : 0.f; }
                    }
                    const int row = r0 + 8 * h;
                    const int boff = cl * ES;
                    uint8_t* dst = sbuf + row * 128 + ((((boff >> 4) ^ (row & 7))) << 4) + (boff & 15);
                    if (CF32) {
                        *reinterpret_cast<float2*>(dst) = make_float2(x[0], x[1]);
                    } else {
                        *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(x[0], x[1]);
                    }
                }
            }
            fence_proxy_async_smem();
            named_bar_sync(bar_stage, 128);
            if (p.c_accumulate) tma_reduce_add_4d_p(&p.c, sbuf, nc0, m0, zb0, zb1, store_pred);
            else tma_store_4d_hint_p(&p.c, sbuf, nc0, m0, zb0, zb1, p.pol_c, store_pred);
            tma_store_commit_p(store_pred);
            ++chunk_ctr;
        }
    }
    if constexpr (EPI == EPI_LSE) {                    // the last tile has no next main loop to hide its sums in
        if (lse_pending) {
#pragma unroll
            for (int t = 0; t < LSE_SLICES; ++t) lse_slice(t);
            lse_finish();
        }
    }
    if (!EW && store_pred) tma_store_wait<0>();
    }
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
    return fn;
}

// Build a rank-4 tiled tensor map with 128B swizzle.  box0 * elem_size must be 128 bytes.
static int make_map(CUtensorMap* out, const pk_view4& v, int is_f32, int box0, int box1, const char* what) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return -3; }
    const int es = is_f32 ? 4 : 2;
    cuuint64_t dims[4];
    cuuint64_t strides[3];
    cuuint32_t box[4] = {(cuuint32_t)box0, (cuuint32_t)box1, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    for (int i = 0; i < 4; ++i) {
        if (v.dim[i] <= 0) { set_last_error("gemm %s: dim[%d]=%lld must be > 0", what, i, (long long)v.dim[i]); return -1; }
        dims[i] = (cuuint64_t)v.dim[i];
    }
    for (int i = 0; i < 3; ++i) {
        long long sb = (long long)v.stride[i] * es;
        if (v.dim[i + 1] == 1 && (sb <= 0 || (sb % 16) != 0)) sb = 16;   // unused dimension: any legal stride
        if (sb <= 0 || (sb % 16) != 0) {
            set_last_error("gemm %s: stride[%d]=%lld elements is not a positive multiple of 16 bytes", what, i,
                           (long long)v.stride[i]);
            return -1;
        }
        strides[i] = (cuuint64_t)sb;
    }
    if ((reinterpret_cast<uintptr_t>(v.ptr) & 15) != 0) { set_last_error("gemm %s: base pointer not 16B aligned", what); return -1; }
    if ((cuuint64_t)box[1] > 256) { set_last_error("gemm %s: box too large", what); return -1; }
    CUresult r = enc(out, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                     const_cast<void*>(v.ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("gemm %s: cuTensorMapEncodeTiled failed with CUresult %d", what, (int)r); return -3; }
    return 0;
}

void count_launch();

// rank-3 bf16 map with 128B swizzle for the attention kernels: dims / strides as cuTensorMapEncodeTiled takes them
int encode_tiled_bf16_3d(CUtensorMap* out, const void* ptr, const unsigned long long (&dims)[3], const unsigned long long (&strides_bytes)[2],
                         const unsigned (&box)[3], const char* what) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return -3; }
    {
        static thread_local bool ctx_ready = false;
        if (!ctx_ready) { PK_CHECK_CUDA(cudaFree(nullptr)); ctx_ready = true; }
    }
    cuuint64_t d[3] = {dims[0], dims[1], dims[2]};
    cuuint64_t st[2] = {strides_bytes[0], strides_bytes[1]};
    cuuint32_t bx[3] = {box[0], box[1], box[2]};
    cuuint32_t es[3] = {1, 1, 1};
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (st[0] % 16) != 0 || (st[1] % 16) != 0) {
        set_last_error("%s: base pointer / strides must be 16-byte aligned", what);
        return -1;
    }
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("%s: cuTensorMapEncodeTiled failed with CUresult %d", what, (int)r); return -3; }
    return 0;
}

template <bool A_MN, bool B_MN, int BN, bool CF32, int EPI>
static int launch_gemm_e(const GemmParams& gp, int workers, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, epi_warps<CF32, EPI>()>;
    auto kern = gemm_wgmma_kernel<A_MN, B_MN, BN, CF32, EPI>;
    static bool configured = false;
    if (!configured) {
        PK_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        configured = true;
    }
    kern<<<workers, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(gp);
    PK_CHECK_LAUNCH();
    count_launch();
    return 0;
}

template <bool A_MN, bool B_MN, int BN, bool CF32>
static int launch_gemm(const GemmParams& gp, int workers, cudaStream_t stream) {
    if (gp.row_lse != nullptr) {
        // the row log-sum-exp epilogue exists for the joint projection's layout only: K-major operands, bf16 C, 256-wide tiles
        if constexpr (!A_MN && !B_MN && BN == 256 && !CF32) return launch_gemm_e<false, false, 256, false, EPI_LSE>(gp, workers, stream);
        set_last_error("gemm: row_lse needs K-major operands, a bf16 C and block_n = 256");
        return -1;
    }
    if (gp.drop_thresh != 0u || gp.aux_mode != PK_AUX_NONE) return launch_gemm_e<A_MN, B_MN, BN, CF32, EPI_FULL>(gp, workers, stream);
    return launch_gemm_e<A_MN, B_MN, BN, CF32, EPI_PLAIN>(gp, workers, stream);
}

template <int BN>
static int dispatch_major(const GemmParams& gp, int a_mn, int b_mn, int workers, cudaStream_t stream) {
    if (gp.c_is_f32) {
        if (!a_mn && !b_mn) return launch_gemm<false, false, BN, true>(gp, workers, stream);
        if (!a_mn && b_mn) return launch_gemm<false, true, BN, true>(gp, workers, stream);
        if (a_mn && !b_mn) return launch_gemm<true, false, BN, true>(gp, workers, stream);
        return launch_gemm<true, true, BN, true>(gp, workers, stream);
    }
    if (!a_mn && !b_mn) return launch_gemm<false, false, BN, false>(gp, workers, stream);
    if (!a_mn && b_mn) return launch_gemm<false, true, BN, false>(gp, workers, stream);
    if (a_mn && !b_mn) return launch_gemm<true, false, BN, false>(gp, workers, stream);
    return launch_gemm<true, true, BN, false>(gp, workers, stream);
}

static uint64_t policy_of(int code) { return code == 1 ? kL2EvictFirst : (code == 2 ? kL2EvictLast : kL2EvictNormal); }

// Tile width for an [M, N] output.  One place, shared by the launch and by pk_gemm_row_lse_parts (the caller sizes the partials
// buffer from it).
static int plan_block_n(long long N, int block_n) { return block_n ? block_n : (N <= 64 ? 64 : (N <= 128 ? 128 : 256)); }

}  // namespace pk

// every row's columns of an N tile belong to one CTA: one partial per N tile
extern "C" int pk_gemm_row_lse_parts(long long M, long long N, int block_n) {
    (void)M;
    const int bn = pk::plan_block_n(N, block_n ? block_n : 256);
    return (int)((N + bn - 1) / bn);
}

extern "C" int pk_gemm_bf16(const pk_gemm_desc* d, void* stream_v) {
    using namespace pk;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    PK_CHECK_ARG(d != nullptr, "null descriptor");
    PK_CHECK_ARG(d->n_pairs >= 1 && d->n_pairs <= PK_GEMM_MAX_PAIRS, "n_pairs out of range");
    PK_CHECK_ARG(d->kz_count >= 1, "kz_count must be >= 1");
    PK_CHECK_ARG(d->c_dtype == PK_F32 || d->c_dtype == PK_BF16, "bad c_dtype");
    PK_CHECK_ARG(!d->c_accumulate || d->c_dtype == PK_F32, "c_accumulate needs an f32 C");
    PK_CHECK_ARG(d->drop_p >= 0.f && d->drop_p < 1.f, "drop_p out of range");
    const long long N = d->c.dim[0], M = d->c.dim[1];
    PK_CHECK_ARG(M > 0 && N > 0, "empty C");
    PK_CHECK_ARG(d->aux == nullptr || d->aux_mode == PK_AUX_NONE || (N % 8 == 0), "aux epilogue needs N % 8 == 0");
    PK_CHECK_ARG(d->block_n == 0 || d->block_n == 64 || d->block_n == 128 || d->block_n == 256, "block_n must be 64, 128 or 256");
    const int bn = plan_block_n(N, d->row_lse ? (d->block_n ? d->block_n : 256) : d->block_n);

    {   // the tensor-map encoder is a driver-API call: make sure this host thread (e.g. an autograd worker) has the primary context bound
        static thread_local bool ctx_ready = false;
        if (!ctx_ready) { PK_CHECK_CUDA(cudaFree(nullptr)); ctx_ready = true; }
    }
    static thread_local GemmParams gp;   // ~2.6 KB; filled per call, copied into the launch
    memset(&gp, 0, sizeof(gp));
    long long K = d->a_mn_major ? d->a[0].dim[1] : d->a[0].dim[0];
    for (int i = 0; i < d->n_pairs; ++i) {
        const long long ka = d->a_mn_major ? d->a[i].dim[1] : d->a[i].dim[0];
        const long long kb = d->b_mn_major ? d->b[i].dim[1] : d->b[i].dim[0];
        PK_CHECK_ARG(ka == K && kb == K, "all pairs must share the reduction extent K");
        int rc = make_map(&gp.a[i], d->a[i], 0, 64, d->a_mn_major ? 64 : BM, "A");
        if (rc) return rc;
        rc = make_map(&gp.b[i], d->b[i], 0, 64, d->b_mn_major ? 64 : bn, "B");
        if (rc) return rc;
        gp.a_off[i] = d->a_row_off[i];
        gp.b_off[i] = d->b_row_off[i];
    }
    {
        int rc = make_map(&gp.c, d->c, d->c_dtype == PK_F32, d->c_dtype == PK_F32 ? 32 : 64, 64, "C");   // one consumer's 64 rows
        if (rc) return rc;
    }
    gp.n_pairs = d->n_pairs;
    gp.kz_count = d->kz_count;
    gp.num_k_blocks = (int)((K + BK - 1) / BK);
    gp.M = (int)M;
    gp.N = (int)N;
    gp.tiles_m = (int)((M + BM - 1) / BM);
    gp.tiles_n = (int)((N + bn - 1) / bn);
    gp.zb0 = (int)d->c.dim[2];
    gp.zb1 = (int)d->c.dim[3];
    gp.a_sel2 = d->a_sel2; gp.a_sel3 = d->a_sel3; gp.b_sel2 = d->b_sel2; gp.b_sel3 = d->b_sel3;
    gp.c_is_f32 = d->c_dtype == PK_F32;
    gp.c_accumulate = d->c_accumulate;
    gp.alpha = d->alpha;
    gp.bias = d->bias;
    gp.act = d->act;
    if (d->drop_p > 0.f) {
        double t = (double)d->drop_p * 4294967296.0;
        gp.drop_thresh = t >= 4294967295.0 ? 4294967295u : (uint32_t)t;
        if (gp.drop_thresh == 0) gp.drop_thresh = 1;
        gp.drop_scale = 1.f / (1.f - d->drop_p);
    }
    gp.drop_seed = d->drop_seed;
    gp.aux_mode = d->aux ? d->aux_mode : PK_AUX_NONE;
    gp.aux_is_f32 = d->aux_dtype == PK_F32;
    gp.aux = d->aux;
    gp.aux_sm = d->aux_stride[0]; gp.aux_s0 = d->aux_stride[1]; gp.aux_s1 = d->aux_stride[2];
    gp.aux_scale = d->aux_scale;
    gp.row_lse = d->row_lse;
    gp.a_rows_dev = d->a_rows_dev;
    PK_CHECK_ARG(d->a_rows_dev == nullptr || (d->n_pairs == 1 && d->kz_count == 1 && gp.zb0 == 1 && gp.zb1 == 1 &&
                                              (d->a_mn_major || d->k_splits <= 1)),
                 "a_rows_dev needs one pair, kz_count 1, a 2-D C and, for a K-major A, no split-K");
    PK_CHECK_ARG(d->row_lse == nullptr || (d->c_dtype == PK_BF16 && N % 8 == 0 && gp.zb0 == 1 && gp.zb1 == 1 && bn == 256 &&
                                           gp.drop_thresh == 0u && gp.aux_mode == PK_AUX_NONE),
                 "row_lse needs a 2-D bf16 C with N % 8 == 0, block_n = 256, no dropout / aux");
    {   // L2 eviction priorities by stream size: an operand that fits in L2 many times over (a weight matrix) is kept with evict_last,
        // a multi-GB streamed operand (the wgrad's activations) is not; a C stream much larger than L2 leaves first.
        const long long K_ = (long long)gp.num_k_blocks * BK * gp.kz_count;
        const long long a_bytes = M * K_ * 2 * gp.n_pairs, b_bytes = N * K_ * 2 * gp.n_pairs;
        const long long c_bytes = M * N * (gp.c_is_f32 ? 4 : 2) * gp.zb0 * gp.zb1;
        const long long small = 32ll << 20, big = 256ll << 20;
        gp.pol_a = policy_of(a_bytes <= small && gp.zb0 * gp.zb1 == 1 ? 2 : 0);
        gp.pol_b = policy_of(b_bytes <= small && gp.zb0 * gp.zb1 == 1 ? 2 : 0);
        gp.pol_c = policy_of(c_bytes >= big ? 1 : 0);
    }

    const long long out_tiles = (long long)gp.tiles_m * gp.tiles_n * gp.zb0 * gp.zb1;
    const int workers_max = num_sms();
    // split-K: under-filled grids with a long reduction (wgrad, the LSTM's recurrent dgrad) are cut along the
    // flattened (pair, kz, k-block) axis; partial tiles are combined with TMA reduce-add into a zeroed f32 C.
    const int k_iters_total = gp.n_pairs * gp.kz_count * gp.num_k_blocks;
    int splits = 1;
    const bool plain_epi = d->bias == nullptr && d->act == PK_ACT_NONE && d->drop_p == 0.f && gp.aux_mode == PK_AUX_NONE;
    if (d->k_splits > 0) splits = d->k_splits;
    else if (gp.c_is_f32 && plain_epi && gp.zb0 == 1 && gp.zb1 == 1 && k_iters_total >= 16 && out_tiles < 6 * workers_max &&
             (d->a_rows_dev == nullptr || d->a_mn_major)) {
        // the split count (>= 8 k-blocks each, <= 16) that wastes the least of the last wave, preferring fewer splits on ties
        const int w = workers_max;
        double best = 0.0;
        for (int sp = 1; sp <= 16 && sp <= k_iters_total / 8; ++sp) {
            const long long units = out_tiles * sp;
            const double eff = (double)units / (double)(((units + w - 1) / w) * w);
            if (eff > best + 0.02) { best = eff; splits = sp; }
        }
    }
    PK_CHECK_ARG(splits == 1 || (gp.c_is_f32 && plain_epi && gp.zb0 == 1 && gp.zb1 == 1), "split-K needs a plain f32 2-D C");
    gp.iters_per_split = (k_iters_total + splits - 1) / splits;
    gp.k_splits = (k_iters_total + gp.iters_per_split - 1) / gp.iters_per_split;
    if (gp.k_splits > 1) {
        if (!gp.c_accumulate)
            PK_CHECK_CUDA(cudaMemset2DAsync(const_cast<void*>(d->c.ptr), (size_t)d->c.stride[0] * 4, 0, (size_t)N * 4, (size_t)M, stream));
        gp.c_accumulate = 1;
    }
    const long long num_tiles = out_tiles * gp.k_splits;
    PK_CHECK_ARG(num_tiles < (1ll << 31), "too many tiles");
    int grid = workers_max;
    if (num_tiles < grid) grid = (int)num_tiles;
    if (bn == 64) return dispatch_major<64>(gp, d->a_mn_major, d->b_mn_major, grid, stream);
    if (bn == 128) return dispatch_major<128>(gp, d->a_mn_major, d->b_mn_major, grid, stream);
    return dispatch_major<256>(gp, d->a_mn_major, d->b_mn_major, grid, stream);
}
