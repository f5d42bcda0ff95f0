// Persistent LSTM layer kernels: the whole time recurrence (forward, and back-propagation through time)
// runs inside ONE cooperative launch instead of two launches per step.
//
// Replaces cuDNN's nn.LSTM recurrence for the prediction net (trainer/model/transducer.py:56-61,95) and for the LSTM encoder
// (:38-44,82-86): ragged lengths (packed sequences), reverse direction, and both directions of a layer in one launch.
//
// Work split: the hidden units are sharded across the CTAs (HJ = 8 units per CTA -> H/8 = 128 CTAs for
// H = 1024, one per SM).  A CTA keeps its slice of the recurrent weights resident in shared memory for all U
// steps: forward the 4*HJ gate rows W_hh[g*H + j, :], backward the transposed columns W_hh[:, j].  Per step
// every CTA reads the full previous hidden state (forward, 64 KB) or the full gate-gradient row block
// (backward, 256 KB) from L2, multiplies it against its resident slice on the tensor cores, applies the fused
// cell update for its (batch, unit) pairs, publishes its slice, and the grid meets at a barrier.
//
// The batch is tiny (<= 32 rows = two m16 tiles) and the op is latency-bound, so the products use the
// warp-level mma.sync.m16n8k16 path: a wgmma tile needs M >= 64 rows per warpgroup and a warpgroup-wide
// issue / wait per step, twice the batch and more latency for no throughput benefit.  (Every throughput-bound contraction
// of the model goes through the wgmma kernel in gemm.cu, including this layer's input projection, dW_ih,
// dW_hh and dx.)  bf16 operands, fp32 accumulation and state.
#include <cooperative_groups.h>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

constexpr int LS_HJ = 8;          // hidden units per CTA
constexpr int LS_MB = 32;         // batch rows per launch
constexpr int LS_THREADS = 256;
constexpr int LS_PAD = 8;         // bf16 elements of row padding (bank-conflict-free fragment loads)

PK_DEVICE void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
PK_DEVICE uint4 ldcg16(const void* p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// 1-D bulk async copy global -> shared (TMA engine, no register staging), completion on an mbarrier
PK_DEVICE void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// same copy delivered to the same shared-memory offset (and signalled on the mbarrier at the same offset) of every CTA in ``mask``
PK_DEVICE void bulk_g2s_mc(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint16_t mask) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
                 : "memory");
}
PK_DEVICE void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Release reduction on the counter, acquire polling loads: this CTA's writes of the step are ordered before its arrival by bar.sync +
// cumulativity, so no separate membar.gl is needed on either side.  (A hierarchical form -- a hardware cluster barrier, one thread per
// cluster doing this handshake on the counter, a second cluster barrier to release the peers -- measured slower: 6.49 against 5.81 us
// per forward step; the two cluster barriers cost more than the contention they remove.)
// ``nct`` = CTAs that meet at this barrier: the CTAs of one direction (a bidirectional launch keeps one counter per direction, so
// the two recurrences never wait on each other).
PK_DEVICE void grid_barrier(unsigned int* counter, unsigned int step_index, unsigned int nct) {
    const unsigned int target = nct * step_index;
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        unsigned int seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
    }
    __syncthreads();
}
PK_DEVICE float sigm(float x) { return 1.f / (1.f + __expf(-x)); }

// Per-launch sequence lengths into len_s[32] (rows >= B get 0; lens == NULL: every row runs all U steps, clamped to [0, U]);
// returns the number of steps of this launch, max_b L_b.  Called by every thread before the first __syncthreads.
PK_DEVICE void load_lens(const int* lens, int B, int U, int* len_s, int* steps_s) {
    if (threadIdx.x < 32) {
        int L = 0;
        if ((int)threadIdx.x < B) L = lens ? min(max(lens[threadIdx.x], 0), U) : U;
        len_s[threadIdx.x] = L;
        int m = L;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) *steps_s = m;
    }
}

// Directions.  A launch of n_dir * H/8 CTAs runs n_dir independent recurrences: CTAs [d*H/8, (d+1)*H/8) are direction d, with
// their own W_hh block, gate buffers, exchange buffer and barrier counter (clusters never straddle two directions: the cluster
// size divides H/8).  Direction 1 of a bidirectional launch, or a single-direction launch with ``reverse`` set, runs backwards in
// time: sequence b with length L_b processes step s at time t = L_b - 1 - s.  The forward direction processes t = s.  Both run only
// while s < L_b, from a zero state.
struct LsDir {
    int d;          // buffer index (0 .. n_dir-1)
    bool rev;       // runs backwards in time
    int j0;         // first hidden unit of this CTA
    unsigned nct;   // CTAs of this direction
};
PK_DEVICE LsDir ls_dir(int H, int reverse) {
    LsDir r;
    r.nct = (unsigned)(H / LS_HJ);
    r.d = (int)(blockIdx.x / r.nct);
    r.rev = gridDim.x > r.nct ? r.d == 1 : reverse != 0;
    r.j0 = (int)(blockIdx.x - r.d * r.nct) * LS_HJ;
    return r;
}

// ------------------------------------------------------------------------------------------ forward
// Per direction d: gx [B,U,4H] f32 (input projection + both biases); w_hh bf16 [4H,H]; out (T) [B,U,ldo], columns [d*H, (d+1)*H);
// hx bf16 [2,32,H] exchange; gates_save f32 [U,B,4H] (post-activation i,f,g,o), cs f32 [U,B,H]; the n_dir blocks of gx, w_hh,
// gates_save, cs and hx are stacked, and the barrier counters are 128 B apart.  Outputs at t >= L_b are written as exact zeros;
// gates_save / cs at those positions are left untouched.
template <typename T>
__global__ void __launch_bounds__(LS_THREADS, 1) lstm_seq_fwd_kernel(const float* __restrict__ gx, const __nv_bfloat16* __restrict__ w_hh,
                                                                     T* __restrict__ out, int ldo, __nv_bfloat16* hx, float* __restrict__ gates_save,
                                                                     float* __restrict__ cs, const int* __restrict__ lens, int B, int Bt, int U,
                                                                     int H, int reverse, unsigned int* counter) {
    // B = sequences of this launch (<= 32); Bt = sequences of the whole batch: gates_save / cs are time-major [U, Bt, .] and the
    // caller passes them already offset to this launch's first sequence (batches larger than 32 run as independent launches)
    extern __shared__ __align__(16) uint8_t sm_raw[];
    const int P = H + LS_PAD;
    __nv_bfloat16* w_s = reinterpret_cast<__nv_bfloat16*>(sm_raw);               // [32][P]: row g*8+jj = W_hh[g*H + j0 + jj]
    __nv_bfloat16* h_s = w_s + 32 * P;                                           // [32][P]: h_{t-1}
    float* g_s = reinterpret_cast<float*>(h_s + 32 * P);                         // [32][33]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const LsDir dir = ls_dir(H, reverse);
    const int j0 = dir.j0;
    gx += (long long)dir.d * Bt * U * 4 * H;
    w_hh += (long long)dir.d * 4 * H * H;
    out += dir.d * H;
    hx += (long long)dir.d * 2 * LS_MB * H;
    gates_save += (long long)dir.d * U * Bt * 4 * H;
    cs += (long long)dir.d * U * Bt * H;
    counter += dir.d * 32;
    __shared__ int len_s[LS_MB], steps_s;
    load_lens(lens, B, U, len_s, &steps_s);
    const int vec_per_row = H / 8;
    for (int i = tid; i < 32 * vec_per_row; i += LS_THREADS) {
        const int r = i / vec_per_row, v = i - r * vec_per_row;
        const int grow = (r >> 3) * H + j0 + (r & 7);
        *reinterpret_cast<uint4*>(w_s + r * P + v * 8) = *reinterpret_cast<const uint4*>(w_hh + (long long)grow * H + v * 8);
    }
    const int cb = tid >> 3, cj = tid & 7;                                      // cell ownership: batch row, local unit
    float c_state = 0.f;
    const int mt = warp & 1, nt = warp >> 1;                                    // 2 m-tiles x 4 n-tiles of the [32 x 32] product
    const int g = lane >> 2, tq = lane & 3;
    __shared__ __align__(8) uint64_t h_bar;
    if (tid == 0) { mbar_init(&h_bar, 1); mbar_fence_init(); }
    uint32_t h_phase = 0;
    const uint32_t cn = cluster_nctarank(), cr = cluster_ctarank();
    const uint16_t cmask = (uint16_t)((1u << cn) - 1u);
    __syncthreads();
    if (cn > 1) cluster_sync_all();                                              // every peer's barrier exists before the first multicast
    const int S = steps_s, L = len_s[cb];
    for (int s = 0; s < S; ++s) {
        const bool active = s < L;
        const int t = dir.rev ? L - 1 - s : s;                                   // this row's time at step s
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        // this step's input-projection terms do not depend on h_{t-1}: fetch them now so that their L2 / HBM latency hides behind the
        // all-gather and the product instead of sitting on the step's critical path
        float gx_i = 0.f, gx_f = 0.f, gx_g = 0.f, gx_o = 0.f;
        if (active) {
            const float* gxr = gx + ((long long)cb * U + t) * 4 * H + j0 + cj;
            gx_i = __ldg(gxr); gx_f = __ldg(gxr + H); gx_g = __ldg(gxr + 2 * H); gx_o = __ldg(gxr + 3 * H);
        }
        if (s > 0) {
            // all-gather of the previous step's h (32 x H bf16) from L2 by the TMA engine: lane r of warp 0 copies row r
            const __nv_bfloat16* src = hx + (long long)((s - 1) & 1) * LS_MB * H;
            // the CTAs of a cluster share the gather: each fetches 32 / cn of the rows and multicasts them to all cn (one L2 read per
            // cluster instead of one per CTA -- with 128 CTAs pulling the same 64 KB every step the L2 was the bottleneck)
            if (warp == 0) {
                fence_proxy_async_all();
                if (lane == 0) mbar_arrive_expect_tx(&h_bar, 32u * (uint32_t)H * 2u);
                __syncwarp();
                if (cn == 1) bulk_g2s(h_s + lane * P, src + (long long)lane * H, (uint32_t)H * 2u, &h_bar);
                else if ((lane % cn) == cr) bulk_g2s_mc(h_s + lane * P, src + (long long)lane * H, (uint32_t)H * 2u, &h_bar, cmask);
            }
            mbar_wait(&h_bar, h_phase);
            h_phase ^= 1;
            const __nv_bfloat16* ar0 = h_s + (mt * 16 + g) * P + 2 * tq;
            const __nv_bfloat16* ar1 = ar0 + 8 * P;
            const __nv_bfloat16* br = w_s + (nt * 8 + g) * P + 2 * tq;
            // four independent accumulator chains: one chain would serialise H/16 = 64 dependent tensor-core instructions per step
            float acc1[4] = {0.f, 0.f, 0.f, 0.f}, acc2[4] = {0.f, 0.f, 0.f, 0.f}, acc3[4] = {0.f, 0.f, 0.f, 0.f};
            auto mma_at = [&](float (&c)[4], int k0) {
                const uint32_t a0 = *reinterpret_cast<const uint32_t*>(ar0 + k0), a1 = *reinterpret_cast<const uint32_t*>(ar1 + k0);
                const uint32_t a2 = *reinterpret_cast<const uint32_t*>(ar0 + k0 + 8), a3 = *reinterpret_cast<const uint32_t*>(ar1 + k0 + 8);
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(br + k0), b1 = *reinterpret_cast<const uint32_t*>(br + k0 + 8);
                mma_bf16_16816(c, a0, a1, a2, a3, b0, b1);
            };
#pragma unroll 4
            for (int k0 = 0; k0 < H; k0 += 64) {
                mma_at(acc, k0);
                mma_at(acc1, k0 + 16);
                mma_at(acc2, k0 + 32);
                mma_at(acc3, k0 + 48);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e] = (acc[e] + acc1[e]) + (acc2[e] + acc3[e]);
        }
        g_s[(mt * 16 + g) * 33 + nt * 8 + 2 * tq] = acc[0];
        g_s[(mt * 16 + g) * 33 + nt * 8 + 2 * tq + 1] = acc[1];
        g_s[(mt * 16 + g + 8) * 33 + nt * 8 + 2 * tq] = acc[2];
        g_s[(mt * 16 + g + 8) * 33 + nt * 8 + 2 * tq + 1] = acc[3];
        __syncthreads();
        // fused cell for (cb, j0 + cj); local gate rows: i = cj, f = 8 + cj, g = 16 + cj, o = 24 + cj
        if (active) {
            const float gi = sigm(g_s[cb * 33 + cj] + gx_i);
            const float gf = sigm(g_s[cb * 33 + 8 + cj] + gx_f);
            const float gg = tanhf(g_s[cb * 33 + 16 + cj] + gx_g);
            const float go = sigm(g_s[cb * 33 + 24 + cj] + gx_o);
            c_state = gf * c_state + gi * gg;
            const float hv = go * tanhf(c_state);
            out[((long long)cb * U + t) * ldo + j0 + cj] = from_f32<T>(hv);
            hx[(long long)(s & 1) * LS_MB * H + (long long)cb * H + j0 + cj] = __float2bfloat16_rn(hv);
            float* gs = gates_save + ((long long)t * Bt + cb) * 4 * H + j0 + cj;
            gs[0] = gi; gs[H] = gf; gs[2 * H] = gg; gs[3 * H] = go;
            cs[((long long)t * Bt + cb) * H + j0 + cj] = c_state;
        } else {
            hx[(long long)(s & 1) * LS_MB * H + (long long)cb * H + j0 + cj] = __float2bfloat16_rn(0.f);
            if (cb < B) out[((long long)cb * U + s) * ldo + j0 + cj] = from_f32<T>(0.f);      // s >= L_b: a padded position
        }
        if (s + 1 < S) grid_barrier(counter, (unsigned int)(s + 1), dir.nct);
    }
    if (cb < B)
        for (int t = S; t < U; ++t) out[((long long)cb * U + t) * ldo + j0 + cj] = from_f32<T>(0.f);     // past this launch's longest sequence
}

// ------------------------------------------------------------------------------------------ backward
// Per direction d: dout (T) [B,U,ldo], columns [d*H, (d+1)*H); gates_save, cs as saved by the forward; w_hh bf16 [4H,H];
// dG bf16 [U,B,4H] (gradient w.r.t. the pre-activation gates, time-major: feeds dW_ih / dW_hh / dx GEMMs).  Rows of dG at
// t >= L_b are written as zeros, so those GEMMs run over all U x B rows unmasked.  zrow: 4H zero bf16 values, the recurrent
// input of a sequence's first backward step.  The recurrent gradient dh_rec = W_hh^T dG_{t+1} is split over four K-groups of warps;
// each stores its partial into its own slot of r_s and the cell adds the four slots in K-group order, so dh_rec (and through
// dc_state every earlier dG) is the same bits on every run.  (Shared-memory atomics in their place gave run-to-run dG differences
// in the last bits.  The fixed order is no slower: 1.53 against 1.57 ms for the B = 32, U = 151, H = 1024 backward, measured on
// an H100 80GB HBM3 at 700 W.)
template <typename T>
__global__ void __launch_bounds__(LS_THREADS, 1) lstm_seq_bwd_kernel(const T* __restrict__ dout, int ldo, const float* __restrict__ gates_save,
                                                                     const float* __restrict__ cs, const __nv_bfloat16* __restrict__ w_hh,
                                                                     __nv_bfloat16* dG, const __nv_bfloat16* zrow, const int* __restrict__ lens,
                                                                     int B, int Bt, int U, int H, int reverse, unsigned int* counter) {
    extern __shared__ __align__(16) uint8_t sm_raw[];
    const int G4 = 4 * H;
    const int PW = G4 + LS_PAD;                                                  // Wt_s pitch
    const int KQ = G4 / 4;                                                       // K quarter per pipeline stage
    const int PD = KQ + LS_PAD;
    __nv_bfloat16* wt_s = reinterpret_cast<__nv_bfloat16*>(sm_raw);              // [8][PW]: wt_s[jj][r] = W_hh[r][j0+jj]
    __nv_bfloat16* d_s = wt_s + LS_HJ * PW;                                      // [2][32][PD]: quarters of dG_{t+1}, double-buffered
    float* r_s = reinterpret_cast<float*>(d_s + 2 * 32 * PD);                    // [4][32][9] dh_rec partial of each K-group
    __shared__ __align__(8) uint64_t q_bar[2];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const LsDir dir = ls_dir(H, reverse);
    const int j0 = dir.j0;
    dout += dir.d * H;
    gates_save += (long long)dir.d * U * Bt * G4;
    cs += (long long)dir.d * U * Bt * H;
    w_hh += (long long)dir.d * G4 * H;
    dG += (long long)dir.d * U * Bt * G4;
    counter += dir.d * 32;
    __shared__ int len_s[LS_MB], steps_s;
    load_lens(lens, B, U, len_s, &steps_s);
    for (int i = tid; i < G4 * LS_HJ; i += LS_THREADS) {
        const int r = i / LS_HJ, jj = i - r * LS_HJ;
        wt_s[jj * PW + r] = w_hh[(long long)r * H + j0 + jj];
    }
    for (int i = tid; i < 2 * 32 * PD / 8; i += LS_THREADS) reinterpret_cast<uint4*>(d_s)[i] = make_uint4(0, 0, 0, 0);   // rows >= B stay zero
    for (int i = tid; i < 4 * 32 * 9; i += LS_THREADS) r_s[i] = 0.f;            // the first step has no product; later steps overwrite every slot
    if (tid == 0) { mbar_init(&q_bar[0], 1); mbar_init(&q_bar[1], 1); mbar_fence_init(); }
    const int cb = tid >> 3, cj = tid & 7;
    float dc_state = 0.f;
    const int mt = warp & 1, kg = warp >> 1;                                     // 2 m-tiles x 4 K-groups
    const int g = lane >> 2, tq = lane & 3;
    uint32_t q_phase[2] = {0, 0};
    const uint32_t cn = cluster_nctarank(), cr = cluster_ctarank();
    const uint16_t cmask = (uint16_t)((1u << cn) - 1u);
    __syncthreads();
    if (cn > 1) cluster_sync_all();                                              // every peer's barriers exist before the first multicast
    const int S = steps_s, L = len_s[cb];
    if (cb < B)
        for (int t = S; t < U; ++t) {                                            // past this launch's longest sequence
            __nv_bfloat16* d = dG + ((long long)t * Bt + cb) * G4 + j0 + cj;
            d[0] = d[H] = d[2 * H] = d[3 * H] = __float2bfloat16_rn(0.f);
        }
    // the recurrent input of row `lane` at step s comes from its step s + 1 (time t + 1 forward, t - 1 backwards in time), or is zero
    // when s + 1 is past its length
    const int Lr = len_s[lane];
    for (int s = S - 1; s >= 0; --s) {
        const bool active = s < L;
        const int t = dir.rev ? L - 1 - s : s;
        // saved forward values of this step: independent of the recurrent gradient, fetched before the product (latency off the critical path)
        float pgi = 0.f, pgf = 0.f, pgg = 0.f, pgo = 0.f, pc = 0.f, pcp = 0.f, pdo = 0.f;
        if (active) {
            const int j = j0 + cj;
            const int tp = dir.rev ? t + 1 : t - 1;                              // the previous step's time
            const float* gs = gates_save + ((long long)t * Bt + cb) * G4 + j;
            pgi = __ldg(gs); pgf = __ldg(gs + H); pgg = __ldg(gs + 2 * H); pgo = __ldg(gs + 3 * H);
            pc = __ldg(cs + ((long long)t * Bt + cb) * H + j);
            pcp = s > 0 ? __ldg(cs + ((long long)tp * Bt + cb) * H + j) : 0.f;
            pdo = to_f32<T>(dout[((long long)cb * U + t) * ldo + j]);
        }
        if (s < S - 1) {
            const int tn = dir.rev ? Lr - 2 - s : s + 1;
            const __nv_bfloat16* src = s + 1 < Lr ? dG + ((long long)tn * Bt + lane) * G4 : zrow;
            auto issue = [&](int qtr) {                                          // warp 0: lane r copies row r of quarter `qtr`
                if (warp == 0) {
                    fence_proxy_async_all();
                    if (lane == 0) mbar_arrive_expect_tx(&q_bar[qtr & 1], (uint32_t)B * (uint32_t)KQ * 2u);
                    __syncwarp();
                    __nv_bfloat16* dst = d_s + ((qtr & 1) * 32 + lane) * PD;
                    const __nv_bfloat16* from = src + qtr * KQ;
                    if (lane < B) {
                        // cluster: each CTA fetches every cn-th row and multicasts it to all cn CTAs (every CTA needs the whole 256 KB
                        // row block each step: one L2 read per cluster instead of one per CTA)
                        if (cn == 1) bulk_g2s(dst, from, (uint32_t)KQ * 2u, &q_bar[qtr & 1]);
                        else if ((lane % cn) == cr) bulk_g2s_mc(dst, from, (uint32_t)KQ * 2u, &q_bar[qtr & 1], cmask);
                    }
                }
            };
            issue(0);
            issue(1);
            float acc[4] = {0.f, 0.f, 0.f, 0.f}, accb[4] = {0.f, 0.f, 0.f, 0.f}, accc[4] = {0.f, 0.f, 0.f, 0.f}, accd[4] = {0.f, 0.f, 0.f, 0.f};
            const int kspan = KQ / 4;                                            // per K-group
            for (int qtr = 0; qtr < 4; ++qtr) {
                mbar_wait(&q_bar[qtr & 1], q_phase[qtr & 1]);
                q_phase[qtr & 1] ^= 1;
                const __nv_bfloat16* ar0 = d_s + ((qtr & 1) * 32 + mt * 16 + g) * PD + kg * kspan + 2 * tq;
                const __nv_bfloat16* ar1 = ar0 + 8 * PD;
                const __nv_bfloat16* br = wt_s + g * PW + qtr * KQ + kg * kspan + 2 * tq;
                auto mma_at = [&](float (&c)[4], int k0) {
                    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(ar0 + k0), a1 = *reinterpret_cast<const uint32_t*>(ar1 + k0);
                    const uint32_t a2 = *reinterpret_cast<const uint32_t*>(ar0 + k0 + 8), a3 = *reinterpret_cast<const uint32_t*>(ar1 + k0 + 8);
                    const uint32_t b0 = *reinterpret_cast<const uint32_t*>(br + k0), b1 = *reinterpret_cast<const uint32_t*>(br + k0 + 8);
                    mma_bf16_16816(c, a0, a1, a2, a3, b0, b1);
                };
                int k0 = 0;
#pragma unroll 4
                for (; k0 + 64 <= kspan; k0 += 64) {
                    mma_at(acc, k0);
                    mma_at(accb, k0 + 16);
                    mma_at(accc, k0 + 32);
                    mma_at(accd, k0 + 48);
                }
                for (; k0 < kspan; k0 += 16) mma_at(acc, k0);                    // kspan = H / 4 is a multiple of 16, not always of 64
                if (qtr + 2 < 4) {
                    if (cn == 1) __syncthreads();                                // every warp is done reading this buffer
                    else cluster_sync_all();                                     // ... in every CTA of the cluster: peers write into it too
                    issue(qtr + 2);
                }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e] = (acc[e] + accb[e]) + (accc[e] + accd[e]);     // four independent tensor-core chains
            float* r_k = r_s + kg * 32 * 9;
            r_k[(mt * 16 + g) * 9 + 2 * tq] = acc[0];
            r_k[(mt * 16 + g) * 9 + 2 * tq + 1] = acc[1];
            r_k[(mt * 16 + g + 8) * 9 + 2 * tq] = acc[2];
            r_k[(mt * 16 + g + 8) * 9 + 2 * tq + 1] = acc[3];
        }
        __syncthreads();
        if (active) {
            const int j = j0 + cj;
            const float gi = pgi, gf = pgf, gg = pgg, go = pgo, c = pc, cp = pcp;
            const float* r_c = r_s + cb * 9 + cj;
            const float dh = pdo + (((r_c[0] + r_c[32 * 9]) + r_c[2 * 32 * 9]) + r_c[3 * 32 * 9]);
            const float tc = tanhf(c);
            const float dc = dh * go * (1.f - tc * tc) + dc_state;
            __nv_bfloat16* d = dG + ((long long)t * Bt + cb) * G4 + j;
            d[0] = __float2bfloat16_rn(dc * gg * gi * (1.f - gi));
            d[H] = __float2bfloat16_rn(dc * cp * gf * (1.f - gf));
            d[2 * H] = __float2bfloat16_rn(dc * gi * (1.f - gg * gg));
            d[3 * H] = __float2bfloat16_rn(dh * tc * go * (1.f - go));
            dc_state = dc * gf;
        } else if (cb < B) {
            __nv_bfloat16* d = dG + ((long long)s * Bt + cb) * G4 + j0 + cj;     // s >= L_b: a padded position
            d[0] = d[H] = d[2 * H] = d[3 * H] = __float2bfloat16_rn(0.f);
        }
        if (s > 0) grid_barrier(counter, (unsigned int)(S - s), dir.nct);
    }
}
}  // namespace pk

using namespace pk;

// cooperative launch with thread-block clusters of ``cs`` CTAs; cs is the largest of 8/4/2 for which the whole grid is co-resident
static int lstm_launch(const void* fn, int grid, int smem, void** args, cudaStream_t st, int* cluster_cache) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(LS_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeCooperative; attr[0].val.cooperative = 1;
    if (*cluster_cache == 0) {
        int pick = 1;
        for (int cs = 8; cs >= 2; cs >>= 1) {
            if (grid % cs) continue;
            attr[1].id = cudaLaunchAttributeClusterDimension; attr[1].val.clusterDim.x = cs; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 2;
            int ncl = 0;
            if (cudaOccupancyMaxActiveClusters(&ncl, fn, &cfg) == cudaSuccess && ncl * cs >= grid) { pick = cs; break; }
            (void)cudaGetLastError();
        }
        *cluster_cache = pick;
    }
    attr[1].id = cudaLaunchAttributeClusterDimension; attr[1].val.clusterDim.x = *cluster_cache; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 2;
    PK_CHECK_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
    return 0;
}
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static int lstm_seq_check(int B, int U, int H, int n_dir, int ldo) {
    PK_CHECK_ARG(B >= 1, "empty batch");
    PK_CHECK_ARG(U >= 1, "U must be >= 1");
    PK_CHECK_ARG(n_dir == 1 || n_dir == 2, "n_dir must be 1 or 2");
    PK_CHECK_ARG(H >= 64 && H % 64 == 0 && n_dir * H / LS_HJ <= num_sms(), "H must be a multiple of 64 with n_dir * H/8 <= #SMs");
    PK_CHECK_ARG(ldo >= n_dir * H, "ldo must be >= n_dir * H");
    return 0;
}
// the cluster size is chosen once per (kernel flavour, n_dir, H): the grid and the shared memory per CTA both enter the occupancy.
// Every grid is a multiple of 8 CTAs per direction, so a cluster of 8, 4 or 2 never straddles two directions.
static int* lstm_cluster_slot(int (*cache)[2][64], int fl, int n_dir, int H) { return &cache[fl][n_dir - 1][(H / 64) & 63]; }

extern "C" long long pk_lstm_seq_workspace_bytes(int H) { return 2ll * LS_MB * H * 2 + 256 + 4ll * H * 2; }

/* ws: pk_lstm_seq_workspace_bytes(n_dir * H): [barrier counters, one per direction, 128 B apart (256 B)]
 *     [hx bf16 n_dir x 2 x 32 x H] [4 * n_dir * H zero bf16 (never written)] */
extern "C" int pk_lstm_seq_fwd_ex(const float* gx, const void* w_hh_bf16, void* out, int out_dtype, int ldo, float* gates_save, float* cs,
                                  const int* lens, int B, int U, int H, int n_dir, int reverse, void* ws, void* stream) {
    int rc = lstm_seq_check(B, U, H, n_dir, ldo);
    if (rc) return rc;
    // W_hh rows are staged with 16-byte loads and the hidden-state exchange in ws is a cp.async.bulk source
    PK_CHECK_ARG(aligned16(w_hh_bf16) && aligned16(ws), "pk_lstm_seq_fwd_ex: w_hh, ws must be 16-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned int* counter = reinterpret_cast<unsigned int*>(ws);
    __nv_bfloat16* hx = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<unsigned char*>(ws) + 256);
    const int smem = 2 * 32 * (H + LS_PAD) * 2 + 32 * 33 * 4;
    const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(w_hh_bf16);
    const void* fn = out_dtype == PK_BF16 ? (const void*)lstm_seq_fwd_kernel<__nv_bfloat16> : (const void*)lstm_seq_fwd_kernel<float>;
    PK_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const size_t es = out_dtype == PK_BF16 ? 2 : 4;
    const int grid = n_dir * H / LS_HJ;
    static int cluster_f[2][2][64] = {};
    for (int b0 = 0; b0 < B; b0 += LS_MB) {                    // sequences are independent: 32 per cooperative launch
        int nb = B - b0 < LS_MB ? B - b0 : LS_MB, Bt = B;
        const float* gx_c = gx + (long long)b0 * U * 4 * H;
        void* out_c = reinterpret_cast<unsigned char*>(out) + (size_t)b0 * U * ldo * es;
        float* gs_c = gates_save + (long long)b0 * 4 * H;
        float* cs_c = cs + (long long)b0 * H;
        const int* lens_c = lens ? lens + b0 : nullptr;
        PK_CHECK_CUDA(cudaMemsetAsync(counter, 0, 256, st));
        void* args[] = {(void*)&gx_c, (void*)&w, (void*)&out_c, (void*)&ldo, (void*)&hx, (void*)&gs_c, (void*)&cs_c, (void*)&lens_c, (void*)&nb,
                        (void*)&Bt, (void*)&U, (void*)&H, (void*)&reverse, (void*)&counter};
        rc = lstm_launch(fn, grid, smem, args, st, lstm_cluster_slot(cluster_f, out_dtype == PK_BF16 ? 0 : 1, n_dir, H));
        if (rc) return rc;
        count_launch();
    }
    return 0;
}
extern "C" int pk_lstm_seq_bwd_ex(const void* dout, int dtype, int ldo, const float* gates_save, const float* cs, const void* w_hh_bf16,
                                  void* dG_bf16, const int* lens, int B, int U, int H, int n_dir, int reverse, void* ws, void* stream) {
    int rc = lstm_seq_check(B, U, H, n_dir, ldo);
    if (rc) return rc;
    // rows of dG and the zero row in ws are cp.async.bulk sources
    PK_CHECK_ARG(aligned16(dG_bf16) && aligned16(ws), "pk_lstm_seq_bwd_ex: dG, ws must be 16-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned int* counter = reinterpret_cast<unsigned int*>(ws);
    const __nv_bfloat16* zrow = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<unsigned char*>(ws) + 256 + 2ll * LS_MB * n_dir * H * 2);
    const int G4 = 4 * H;
    const int smem = LS_HJ * (G4 + LS_PAD) * 2 + 2 * 32 * (G4 / 4 + LS_PAD) * 2 + 4 * 32 * 9 * 4;     // H = 1024: 202,368 B
    const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(w_hh_bf16);
    const void* fn = dtype == PK_BF16 ? (const void*)lstm_seq_bwd_kernel<__nv_bfloat16> : (const void*)lstm_seq_bwd_kernel<float>;
    PK_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const size_t es = dtype == PK_BF16 ? 2 : 4;
    const int grid = n_dir * H / LS_HJ;
    static int cluster_b[2][2][64] = {};
    for (int b0 = 0; b0 < B; b0 += LS_MB) {
        int nb = B - b0 < LS_MB ? B - b0 : LS_MB, Bt = B;
        const void* dout_c = reinterpret_cast<const unsigned char*>(dout) + (size_t)b0 * U * ldo * es;
        const float* gs_c = gates_save + (long long)b0 * G4;
        const float* cs_c = cs + (long long)b0 * H;
        __nv_bfloat16* dg = reinterpret_cast<__nv_bfloat16*>(dG_bf16) + (long long)b0 * G4;
        const int* lens_c = lens ? lens + b0 : nullptr;
        PK_CHECK_CUDA(cudaMemsetAsync(counter, 0, 256, st));
        void* args[] = {(void*)&dout_c, (void*)&ldo, (void*)&gs_c, (void*)&cs_c, (void*)&w, (void*)&dg, (void*)&zrow, (void*)&lens_c, (void*)&nb,
                        (void*)&Bt, (void*)&U, (void*)&H, (void*)&reverse, (void*)&counter};
        rc = lstm_launch(fn, grid, smem, args, st, lstm_cluster_slot(cluster_b, dtype == PK_BF16 ? 0 : 1, n_dir, H));
        if (rc) return rc;
        count_launch();
    }
    return 0;
}
