// RNN-T loss (alpha/beta lattice) + gradient w.r.t. the joint logits, fused with log-softmax.
//
// Replaces  F.log_softmax (trainer/model/transducer.py:110-111)  +  warp_rnnt.RNNTLoss.apply
// (trainer/train_transducer_bmuf_otfaug.py:58,97-99) and their autograd backward.
//
//   pass 1  rnnt_rowstats   one warp per joint node (b,t,u): streams the V logits once (16-byte
//                           coalesced loads, several in flight per lane), online log-sum-exp ->
//                           lse[b,t,u], lp_blank, lp_label written in a diagonal-major ("skewed")
//                           layout so that pass 2 reads each anti-diagonal contiguously.
//   pass 2  rnnt_lattice    one CTA per utterance: one thread group sweeps alpha, a second one beta
//                           (anti-diagonal wavefront, one lattice cell per thread, previous diagonal
//                           staged in shared memory, next diagonal's log-probs prefetched, fp64);
//                           then all threads emit the per-node gradient coefficients.  Never touches V.
//   pass 3  rnnt_grad       one warp per node: re-reads the logits row and writes
//                           dlogits = -softmax * (gb + gl) + [v==blank] gb + [v==label] gl
//                           (in place if dlogits aliases logits).
// Algorithmic HBM traffic: 3 * B*T*(U+1)*V * sizeof(elem)  (+ O(nodes) fp32).
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <typename T> struct Vec16;
template <> struct Vec16<__nv_bfloat16> {
    static constexpr int N = 8;
    PK_DEVICE static void unpack(const uint4& q, float (&f)[8]) {
        f[0] = bf16lo(q.x); f[1] = bf16hi(q.x); f[2] = bf16lo(q.y); f[3] = bf16hi(q.y);
        f[4] = bf16lo(q.z); f[5] = bf16hi(q.z); f[6] = bf16lo(q.w); f[7] = bf16hi(q.w);
    }
    PK_DEVICE static uint4 pack(const float (&f)[8]) {
        return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
    }
    PK_DEVICE static float vmax(const uint4& q) {         // packed bf16x2 max: 3 + 1 instructions for 8 elements
        const __nv_bfloat162 a = __hmax2(*reinterpret_cast<const __nv_bfloat162*>(&q.x), *reinterpret_cast<const __nv_bfloat162*>(&q.y));
        const __nv_bfloat162 b = __hmax2(*reinterpret_cast<const __nv_bfloat162*>(&q.z), *reinterpret_cast<const __nv_bfloat162*>(&q.w));
        const __nv_bfloat162 c = __hmax2(a, b);
        return fmaxf(__low2float(c), __high2float(c));
    }
};
template <> struct Vec16<float> {
    static constexpr int N = 4;
    PK_DEVICE static void unpack(const uint4& q, float (&f)[4]) {
        f[0] = __uint_as_float(q.x); f[1] = __uint_as_float(q.y); f[2] = __uint_as_float(q.z); f[3] = __uint_as_float(q.w);
    }
    PK_DEVICE static uint4 pack(const float (&f)[4]) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
    }
    PK_DEVICE static float vmax(const uint4& q) {
        return fmaxf(fmaxf(__uint_as_float(q.x), __uint_as_float(q.y)), fmaxf(__uint_as_float(q.z), __uint_as_float(q.w)));
    }
};

PK_DEVICE uint4 ld_stream(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
PK_DEVICE uint4 ld_plain(const uint4* p) { return *p; }
PK_DEVICE void st_stream(uint4* p, const uint4& v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

struct RnntDims {
    int B, T, U1, V, ldv;     // padded batch dims; ldv = row pitch of logits in elements
    int ld_labels;
    int ND;                   // T + U1 - 1 diagonals
};
PK_DEVICE size_t skew_index(const RnntDims& d, int b, int t, int u) { return ((size_t)b * d.ND + (t + u)) * d.U1 + u; }

constexpr int ROWSTATS_UNROLL = 4;

// ------------------------------------------------------------------------------------ pass 1
template <typename T>
__global__ void __launch_bounds__(256) rnnt_rowstats_kernel(const T* __restrict__ logits, const int* __restrict__ labels,
                                                            const int* __restrict__ frame_lens, const int* __restrict__ label_lens,
                                                            RnntDims d, float* __restrict__ lse_out, float* __restrict__ lpb_skew,
                                                            float* __restrict__ lpl_skew) {
    constexpr int VN = Vec16<T>::N;
    const int lane = threadIdx.x & 31;
    const long long warp_global = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long rows = (long long)d.B * d.T * d.U1;
    const int nvec = (d.V + VN - 1) / VN;
    for (long long row = warp_global; row < rows; row += n_warps) {
        const int u = (int)(row % d.U1);
        const long long bt = row / d.U1;
        const int t = (int)(bt % d.T);
        const int b = (int)(bt / d.T);
        const int Tn = frame_lens[b], Un = label_lens[b];
        if (t >= Tn || u > Un) continue;       // padded node: never read (warp-uniform)
        const T* rp = logits + row * (long long)d.ldv;
        const uint4* vp = reinterpret_cast<const uint4*>(rp);
        float m = -INFINITY, s = 0.f;          // running max (in log2 units) and sum of 2^(x*log2e - m)
        const int nfull = d.V / VN;            // vectors without a tail; the (rare) partial vector is handled after the loop
        for (int i0 = lane; i0 < nfull; i0 += 32 * ROWSTATS_UNROLL) {
            uint4 q[ROWSTATS_UNROLL];
#pragma unroll
            for (int k = 0; k < ROWSTATS_UNROLL; ++k) {
                const int i = i0 + k * 32;
                if (i < nfull) q[k] = ld_stream(vp + i);
            }
#pragma unroll
            for (int k = 0; k < ROWSTATS_UNROLL; ++k) {
                const int i = i0 + k * 32;
                if (i < nfull) {
                    const float cm = Vec16<T>::vmax(q[k]) * kLog2e;
                    if (cm > m) { s *= exp2f(m - cm); m = cm; }   // rare after the first chunks
                    float f[VN];
                    Vec16<T>::unpack(q[k], f);
#pragma unroll
                    for (int e = 0; e < VN; ++e) s += ex2_approx(fmaf(f[e], kLog2e, -m));   // raw MUFU.EX2: no denormal fix-up sequence
                }
            }
        }
        if (nfull * VN < d.V && lane == 0) {   // partial last vector (V not a multiple of 16 bytes)
            for (int v = nfull * VN; v < d.V; ++v) {
                const float x = to_f32<T>(rp[v]) * kLog2e;
                if (x > m) { s *= exp2f(m - x); m = x; }
                s += exp2f(x - m);
            }
        }
        // combine the 32 lane-local (m, s) pairs
        const float mw = warp_max(m);
        s = (m == -INFINITY) ? 0.f : s * exp2f(m - mw);
        s = warp_sum(s);
        if (lane == 0) {
            const float lse = (mw + log2f(s)) * kLn2;
            const float zb = to_f32<T>(rp[0]);
            lse_out[row] = lse;
            const size_t sk = skew_index(d, b, t, u);
            lpb_skew[sk] = zb - lse;
            if (u < Un) {
                const int y = labels[(size_t)b * d.ld_labels + u];
                lpl_skew[sk] = to_f32<T>(rp[y]) - lse;
            }
        }
    }
}

// ------------------------------------------------------------------------------------ pass 1, fused variant
// The producing GEMM already reduced every logits row to per-N-tile (max, sum) pairs (pk_gemm_desc.row_lse);
// this kernel only merges the n_parts pairs of a row and gathers the blank / label logits: ~100 bytes per row
// instead of a full read of the row.
template <typename T>
__global__ void __launch_bounds__(256) rnnt_rowfinish_kernel(const T* __restrict__ logits, const int* __restrict__ labels,
                                                             const int* __restrict__ frame_lens, const int* __restrict__ label_lens,
                                                             RnntDims d, const float2* __restrict__ parts, int n_parts,
                                                             float* __restrict__ lse_out, float* __restrict__ lpb_skew,
                                                             float* __restrict__ lpl_skew) {
    const long long rows = (long long)d.B * d.T * d.U1;
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < rows; row += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(row % d.U1);
        const long long bt = row / d.U1;
        const int t = (int)(bt % d.T);
        const int b = (int)(bt / d.T);
        const int Tn = frame_lens[b], Un = label_lens[b];
        if (t >= Tn || u > Un) continue;
        float m = -INFINITY;
        for (int i = 0; i < n_parts; ++i) m = fmaxf(m, parts[(size_t)i * rows + row].x);
        float sum = 0.f;
        for (int i = 0; i < n_parts; ++i) {
            const float2 ps = parts[(size_t)i * rows + row];
            sum += ps.y * exp2f(ps.x - m);
        }
        const float lse = (m + log2f(sum)) * kLn2;
        const T* rp = logits + row * (long long)d.ldv;
        lse_out[row] = lse;
        const size_t sk = skew_index(d, b, t, u);
        lpb_skew[sk] = to_f32<T>(rp[0]) - lse;
        if (u < Un) {
            const int y = labels[(size_t)b * d.ld_labels + u];
            lpl_skew[sk] = to_f32<T>(rp[y]) - lse;
        }
    }
}

// ------------------------------------------------------------------------------------ pass 2
// The lattice runs in double precision: alpha/beta reach magnitudes of (T+U)*log V ~ 3000 where an
// fp32 ulp (2.4e-4) would show up as a 1e-4-level relative error in the gradients.  The DP touches
// only O(T*U) values per utterance, so fp64 costs nothing measurable next to the V-axis passes.
typedef double lat_t;
#define LAT_NEG_INF (-(double)INFINITY)
PK_DEVICE lat_t lse2(lat_t a, lat_t b) {
    const lat_t mx = fmax(a, b), mn = fmin(a, b);
    if (mx == LAT_NEG_INF) return LAT_NEG_INF;
    return mx + log1p(exp(mn - mx));
}

// One CTA per utterance, 2*G threads: threads [0,G) sweep alpha over ascending anti-diagonals,
// threads [G,2G) sweep beta over descending ones; thread j owns label positions u = j, j+G, ...
// The previous diagonal lives in shared memory (ping-pong), each group synchronises with its own
// named barrier, and the log-probs of the NEXT diagonal are prefetched before the barrier so the
// L2 latency overlaps the dependent LSE chain.
constexpr int LAT_MAX_G = 512;
constexpr int LAT_MAX_CPT = 4;      // cells per thread => U1 <= 2048

// Emission regularisation (DESIGN.md "FastEmit and delay penalty"), compiled in only when REG: every label arc (t, u) -> (t, u+1)
// gets lam_d * ((T_b - 1)/2 - t) added to its log-prob where the sweeps read it (the tables are left as they are), and the label
// coefficient gl is multiplied by fe_scale = 1 + lambda_fastemit where it is written.  REG = false is the plain lattice.
PK_DEVICE lat_t delay_term(lat_t lam_d, int T, int t) { return lam_d * (0.5 * (lat_t)(T - 1) - (lat_t)t); }

template <bool REG>
__global__ void __launch_bounds__(2 * LAT_MAX_G) rnnt_lattice_kernel(
    const int* __restrict__ frame_lens, const int* __restrict__ label_lens, RnntDims d, int G, int cpt,
    const float* __restrict__ lpb_skew, const float* __restrict__ lpl_skew, lat_t* __restrict__ alpha_skew,
    lat_t* __restrict__ beta_skew, const float* __restrict__ grad_scale, float* __restrict__ costs,
    float* __restrict__ gb_out, float* __restrict__ gl_out, lat_t lam_d, float fe_scale) {
    extern __shared__ lat_t sm[];            // 2 groups x 2 diagonals x (U1 + 2)
    const int b = blockIdx.x;
    const int grp = threadIdx.x >= G ? 1 : 0;
    const int j = threadIdx.x - grp * G;
    const int T = frame_lens[b], U = label_lens[b];
    const int W = d.U1 + 2;
    lat_t* buf0 = sm + grp * 2 * W + 1;      // index -1 .. U1 valid
    lat_t* buf1 = buf0 + W;
    __shared__ lat_t s_ll;
    const size_t base = (size_t)b * d.ND * d.U1;
    const bool valid = (T > 0 && T <= d.T && U >= 0 && U < d.U1);
    if (valid) {
        for (int i = j - 1; i <= d.U1; i += G) { buf0[i] = LAT_NEG_INF; buf1[i] = LAT_NEG_INF; }
        named_bar_sync(1 + grp, G);
        const int last = T - 1 + U;           // last diagonal
        if (grp == 0) {
            // ---------------- alpha: diagonals ascending
            lat_t* prev = buf0;
            lat_t* cur = buf1;
            if (j == 0) { cur[0] = 0.0; alpha_skew[base] = 0.0; }
            float nb[LAT_MAX_CPT], nl[LAT_MAX_CPT];   // lpb(d-1,u), lpl(d-1,u-1) for the upcoming diagonal
#pragma unroll
            for (int c = 0; c < LAT_MAX_CPT; ++c) {
                const int u = j + c * G;
                nb[c] = (c < cpt && u <= U && last >= 1) ? lpb_skew[base + u] : 0.f;
                nl[c] = (c < cpt && u >= 1 && u <= U && last >= 1) ? lpl_skew[base + u - 1] : 0.f;
            }
            named_bar_sync(1, G);
            for (int dg = 1; dg <= last; ++dg) {
                lat_t* tsw = prev; prev = cur; cur = tsw;
                const int lo = max(0, dg - (T - 1)), hi = min(U, dg);
                float pb[LAT_MAX_CPT], pl[LAT_MAX_CPT];
#pragma unroll
                for (int c = 0; c < LAT_MAX_CPT; ++c) { pb[c] = nb[c]; pl[c] = nl[c]; }
                if (dg < last) {                       // prefetch diagonal dg (used at dg+1)
                    const size_t nbase = base + (size_t)dg * d.U1;
#pragma unroll
                    for (int c = 0; c < LAT_MAX_CPT; ++c) {
                        const int u = j + c * G;
                        if (c < cpt && u <= U) {
                            nb[c] = lpb_skew[nbase + u];
                            nl[c] = (u >= 1) ? lpl_skew[nbase + u - 1] : 0.f;
                        }
                    }
                }
#pragma unroll
                for (int c = 0; c < LAT_MAX_CPT; ++c) {
                    const int u = j + c * G;
                    if (c < cpt && u >= lo && u <= hi) {
                        lat_t a = LAT_NEG_INF, cc = LAT_NEG_INF;
                        if (u <= dg - 1) a = prev[u] + pb[c];              // from (t-1, u) via blank
                        if (u >= 1) {                                      // from (t, u-1) via label u, t = dg - u
                            if (REG) cc = prev[u - 1] + ((lat_t)pl[c] + delay_term(lam_d, T, dg - u));
                            else cc = prev[u - 1] + pl[c];
                        }
                        const lat_t v = lse2(a, cc);
                        cur[u] = v;
                        alpha_skew[base + (size_t)dg * d.U1 + u] = v;
                    }
                }
                named_bar_sync(1, G);
            }
        } else {
            // ---------------- beta: diagonals descending
            lat_t* prev = buf0;
            lat_t* cur = buf1;
            if (j == 0) {
                const lat_t v = lpb_skew[base + (size_t)last * d.U1 + U];
                cur[U] = v;
                beta_skew[base + (size_t)last * d.U1 + U] = v;
            }
            float nb[LAT_MAX_CPT], nl[LAT_MAX_CPT];   // lpb(d,u), lpl(d,u) of the upcoming diagonal
#pragma unroll
            for (int c = 0; c < LAT_MAX_CPT; ++c) {
                const int u = j + c * G;
                const bool ok = c < cpt && u <= U && last >= 1;
                nb[c] = ok ? lpb_skew[base + (size_t)(last - 1) * d.U1 + u] : 0.f;
                nl[c] = ok ? lpl_skew[base + (size_t)(last - 1) * d.U1 + u] : 0.f;
            }
            named_bar_sync(2, G);
            for (int dg = last - 1; dg >= 0; --dg) {
                lat_t* tsw = prev; prev = cur; cur = tsw;
                const int lo = max(0, dg - (T - 1)), hi = min(U, dg);
                float pb[LAT_MAX_CPT], pl[LAT_MAX_CPT];
#pragma unroll
                for (int c = 0; c < LAT_MAX_CPT; ++c) { pb[c] = nb[c]; pl[c] = nl[c]; }
                if (dg > 0) {
                    const size_t nbase = base + (size_t)(dg - 1) * d.U1;
#pragma unroll
                    for (int c = 0; c < LAT_MAX_CPT; ++c) {
                        const int u = j + c * G;
                        if (c < cpt && u <= U) { nb[c] = lpb_skew[nbase + u]; nl[c] = lpl_skew[nbase + u]; }
                    }
                }
#pragma unroll
                for (int c = 0; c < LAT_MAX_CPT; ++c) {
                    const int u = j + c * G;
                    if (c < cpt && u >= lo && u <= hi) {
                        const int t = dg - u;
                        lat_t a = LAT_NEG_INF, cc = LAT_NEG_INF;
                        if (t + 1 <= T - 1) a = prev[u] + pb[c];            // to (t+1, u) via blank
                        if (u + 1 <= U) {                                   // to (t, u+1) via label u+1
                            if (REG) cc = prev[u + 1] + ((lat_t)pl[c] + delay_term(lam_d, T, t));
                            else cc = prev[u + 1] + pl[c];
                        }
                        const lat_t v = lse2(a, cc);
                        cur[u] = v;
                        beta_skew[base + (size_t)dg * d.U1 + u] = v;
                    }
                }
                named_bar_sync(2, G);
            }
            if (j == 0) { s_ll = cur[0]; costs[b] = (float)(-cur[0]); }
        }
    } else if (threadIdx.x == 0) {
        costs[b] = 0.f;
    }
    __syncthreads();
    if (gb_out == nullptr) return;             // costs only (pk_rnnt_lattice_costs)
    // ---------------- per-node gradient coefficients (natural [b,t,u] layout); zero for padded nodes
    const float gs = grad_scale ? grad_scale[b] : 1.f;
    const lat_t ll = valid ? s_ll : 0.0;
    const int nodes = d.T * d.U1;
    for (int i = threadIdx.x; i < nodes; i += blockDim.x) {
        const int t = i / d.U1, u = i - t * d.U1;
        float gb = 0.f, gl = 0.f;
        if (valid && t < T && u <= U) {
            const size_t sk = skew_index(d, b, t, u);
            const lat_t a = alpha_skew[sk];
            lat_t bn;
            if (t < T - 1) bn = beta_skew[skew_index(d, b, t + 1, u)];
            else bn = (u == U) ? 0.0 : LAT_NEG_INF;
            gb = (float)(-exp(a + bn + (lat_t)lpb_skew[sk] - ll)) * gs;
            if (u < U) {
                if (REG) {
                    const lat_t lpl = (lat_t)lpl_skew[sk] + delay_term(lam_d, T, t);
                    gl = (float)(-exp(a + beta_skew[skew_index(d, b, t, u + 1)] + lpl - ll)) * gs * fe_scale;
                } else {
                    gl = (float)(-exp(a + beta_skew[skew_index(d, b, t, u + 1)] + (lat_t)lpl_skew[sk] - ll)) * gs;
                }
            }
            if (!(gb == gb)) gb = 0.f;
            if (!(gl == gl)) gl = 0.f;
        }
        gb_out[(size_t)b * nodes + i] = gb;
        gl_out[(size_t)b * nodes + i] = gl;
    }
}

// ------------------------------------------------------------------------------------ forced alignment (pk_rnnt_viterbi)
// The max-plus form of the alpha sweep above, same launch shape (one CTA per utterance, thread j owning u = j, j+G, ..., the previous
// diagonal ping-ponged in shared memory, the next diagonal's log-probs prefetched before the barrier), in f64:
//   delta(0,0) = 0,  delta(t,u) = max(delta(t-1,u) + lpb(t-1,u), delta(t,u-1) + lpl(t,u-1)),
//   score = delta(T-1,U) + lpb(T-1,U).
// The label arc is taken only when it is strictly greater (ties and -inf on both arcs go to blank).  Each node's choice is one bit,
// packed 32 label positions per word by __ballot_sync into dec [B][T+U1-1][ceil(U1/32)] (words whose first u is past U are not
// written).  Then warp 0 walks the bits back from (T-1, U) and writes emit[b][u-1] = t for every label arc: lane k loads the words of
// diagonal dg-k that can hold the path (u-k .. u spans at most two words), so one round of loads serves 32 steps of the walk.
__global__ void __launch_bounds__(LAT_MAX_G) rnnt_viterbi_kernel(const int* __restrict__ frame_lens, const int* __restrict__ label_lens,
                                                               RnntDims d, int G, int cpt, const float* __restrict__ lpb_skew,
                                                               const float* __restrict__ lpl_skew, unsigned* __restrict__ dec,
                                                               float* __restrict__ score, int* __restrict__ emit, int ld_emit) {
    extern __shared__ lat_t sm[];            // 2 diagonals x (U1 + 2)
    __shared__ lat_t s_score;
    const int b = blockIdx.x;
    const int j = threadIdx.x;
    const int T = frame_lens[b], U = label_lens[b];
    const int NW = (d.U1 + 31) / 32;
    const size_t base = (size_t)b * d.ND * d.U1;
    unsigned* db = dec + (size_t)b * d.ND * NW;
    int* eb = emit + (size_t)b * ld_emit;
    const bool valid = (T > 0 && T <= d.T && U >= 0 && U < d.U1);
    if (!valid) {                            // no lattice: no path
        for (int i = j; i < ld_emit; i += G) eb[i] = -1;
        if (j == 0) score[b] = -INFINITY;
        return;
    }
    const int W = d.U1 + 2;
    lat_t* prev = sm + 1;                    // index -1 .. U1 valid
    lat_t* cur = prev + W;
    for (int i = j - 1; i <= d.U1; i += G) { prev[i] = LAT_NEG_INF; cur[i] = LAT_NEG_INF; }
    __syncthreads();
    const int last = T - 1 + U;
    if (j == 0) cur[0] = 0.0;
    for (int w = j; w <= U / 32; w += G) db[w] = 0u;   // diagonal 0: node (0, 0) has no incoming arc
    float nb[LAT_MAX_CPT], nl[LAT_MAX_CPT];
#pragma unroll
    for (int c = 0; c < LAT_MAX_CPT; ++c) {
        const int u = j + c * G;
        nb[c] = (c < cpt && u <= U && last >= 1) ? lpb_skew[base + u] : 0.f;
        nl[c] = (c < cpt && u >= 1 && u <= U && last >= 1) ? lpl_skew[base + u - 1] : 0.f;
    }
    __syncthreads();
    for (int dg = 1; dg <= last; ++dg) {
        lat_t* tsw = prev; prev = cur; cur = tsw;
        const int lo = max(0, dg - (T - 1)), hi = min(U, dg);
        float pb[LAT_MAX_CPT], pl[LAT_MAX_CPT];
#pragma unroll
        for (int c = 0; c < LAT_MAX_CPT; ++c) { pb[c] = nb[c]; pl[c] = nl[c]; }
        if (dg < last) {
            const size_t nbase = base + (size_t)dg * d.U1;
#pragma unroll
            for (int c = 0; c < LAT_MAX_CPT; ++c) {
                const int u = j + c * G;
                if (c < cpt && u <= U) {
                    nb[c] = lpb_skew[nbase + u];
                    nl[c] = (u >= 1) ? lpl_skew[nbase + u - 1] : 0.f;
                }
            }
        }
        unsigned* drow = db + (size_t)dg * NW;
#pragma unroll
        for (int c = 0; c < LAT_MAX_CPT; ++c) {
            if (c < cpt) {                                         // block-uniform: every lane reaches the ballot
                const int u = j + c * G;
                bool lab = false;
                if (u >= lo && u <= hi) {
                    const lat_t a = (u <= dg - 1) ? prev[u] + pb[c] : LAT_NEG_INF;    // from (t-1, u) via blank
                    const lat_t l = (u >= 1) ? prev[u - 1] + pl[c] : LAT_NEG_INF;     // from (t, u-1) via label u
                    lab = l > a;
                    cur[u] = lab ? l : a;
                }
                const unsigned bits = __ballot_sync(0xffffffffu, lab);
                const int u0 = c * G + (j & ~31);                  // G is a multiple of 32: the warp's 32 u are one word
                if ((j & 31) == 0 && u0 <= U) drow[u0 >> 5] = bits;
            }
        }
        __syncthreads();
    }
    if (j == 0) {
        const lat_t s = cur[U] + (lat_t)lpb_skew[base + (size_t)last * d.U1 + U];
        s_score = s;
        score[b] = (float)s;
    }
    __syncthreads();                         // also publishes every warp's decision words to warp 0
    if (j >= 32) return;
    const int lane = j;
    const bool found = s_score != LAT_NEG_INF;
    for (int i = (found ? U : 0) + lane; i < ld_emit; i += 32) eb[i] = -1;
    if (!found) return;
    int t = T - 1, u = U;
    while (t + u > 0) {
        const int dg = t + u;
        const int steps = min(32, dg);                              // diagonals dg .. dg-steps+1; the walk stops at diagonal 0
        unsigned whi = 0u, wlo = 0u;
        if (lane < steps) {
            const unsigned* row = db + (size_t)(dg - lane) * NW;
            whi = row[u >> 5];
            wlo = row[max(u - lane, 0) >> 5];
        }
        const int uw = u >> 5;
        for (int s = 0; s < steps; ++s) {                           // the node (t, u) lies on diagonal dg - s
            const unsigned wh = __shfl_sync(0xffffffffu, whi, s);
            const unsigned wl = __shfl_sync(0xffffffffu, wlo, s);
            const unsigned word = (u >> 5) == uw ? wh : wl;
            if ((word >> (u & 31)) & 1u) {
                if (lane == 0) eb[u - 1] = t;
                --u;
            } else {
                --t;
            }
        }
    }
}

// ------------------------------------------------------------------------------------ row compaction
// Every entry of a row's gradient, -softmax * (gb + gl) plus gb / gl in the blank / label column, is at most |gb| + |gl| in
// magnitude (gb and gl share a sign).  When |gb| + |gl| < 2^-136 every entry is below 2^-134 -- half the smallest bf16 subnormal,
// with room for the f32 rounding of the products -- and the stored bf16 row is all +-0: the row adds nothing to the fc2 dgrad,
// wgrad or bias gradient.  Both terms are then f32 subnormals, whose bit patterns are proportional to their values, so the test
// is an integer sum of the magnitude bits and does not depend on how the compiler treats subnormal arithmetic.
PK_DEVICE bool grad_row_kept(float gb, float gl) {
    return (__float_as_uint(gb) & 0x7fffffffu) + (__float_as_uint(gl) & 0x7fffffffu) >= 0x2000u;   // 0x2000 = 2^-136 as a subnormal
}

// map[r] = index of row r among the kept rows (ascending, so kept rows stay in (b, t, u) order), or -1.  Three launches: kept rows
// per SCAN_TILE-row tile, an exclusive scan of the tile counts in one CTA, then the map.
constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_PER_THREAD = 4;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_PER_THREAD;

PK_DEVICE int block_exclusive_scan(int v, int* s_warp, int* total) {   // SCAN_THREADS threads; s_warp: 32 ints
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
        int s = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        s_warp[lane] = s;                                   // inclusive warp totals
    }
    __syncthreads();
    const int r = x - v + (w > 0 ? s_warp[w - 1] : 0);
    *total = s_warp[31];
    __syncthreads();                                        // s_warp may be reused by the caller's next scan
    return r;
}

PK_DEVICE int tile_kept(const float* gb, const float* gl, long long rows, long long r0, bool (&keep)[SCAN_PER_THREAD]) {
    int n = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; ++k) {
        const long long r = r0 + (long long)threadIdx.x * SCAN_PER_THREAD + k;
        keep[k] = r < rows && grad_row_kept(gb[r], gl[r]);
        n += keep[k];
    }
    return n;
}

__global__ void __launch_bounds__(SCAN_THREADS) grad_rows_count_kernel(const float* __restrict__ gb, const float* __restrict__ gl,
                                                                       long long rows, int* __restrict__ tile_count) {
    __shared__ int s_warp[32];
    bool keep[SCAN_PER_THREAD];
    int total;
    block_exclusive_scan(tile_kept(gb, gl, rows, (long long)blockIdx.x * SCAN_TILE, keep), s_warp, &total);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
}

// exclusive scan of the tile counts in place, *count = kept rows; then zero the rows [count, count rounded up to 64) of dz_c and h_c,
// which the wgrad's last 64-row k-block reads
template <typename T>
__global__ void __launch_bounds__(SCAN_THREADS) grad_rows_scan_kernel(int* __restrict__ tile_count, int n_tiles, int* __restrict__ count,
                                                                      long long rows, T* dz_c, int ldv, T* h_c, int H) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n_tiles; i0 += SCAN_THREADS) {
        const int i = i0 + threadIdx.x;
        const int v = i < n_tiles ? tile_count[i] : 0;
        int total;
        const int ex = block_exclusive_scan(v, s_warp, &total);
        if (i < n_tiles) tile_count[i] = s_carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += total;
        __syncthreads();
    }
    const long long kept = s_carry;
    if (threadIdx.x == 0) *count = (int)kept;
    const long long tail = min(rows, (kept + 63) / 64 * 64);
    for (long long r = kept; r < tail; ++r) {
        for (int c = threadIdx.x; c < ldv; c += SCAN_THREADS) dz_c[r * ldv + c] = from_f32<T>(0.f);
        for (int c = threadIdx.x; c < H; c += SCAN_THREADS) h_c[r * H + c] = from_f32<T>(0.f);
    }
}

__global__ void __launch_bounds__(SCAN_THREADS) grad_rows_map_kernel(const float* __restrict__ gb, const float* __restrict__ gl,
                                                                     long long rows, const int* __restrict__ tile_off, int* __restrict__ map) {
    __shared__ int s_warp[32];
    bool keep[SCAN_PER_THREAD];
    const long long r0 = (long long)blockIdx.x * SCAN_TILE;
    int total;
    int idx = tile_off[blockIdx.x] + block_exclusive_scan(tile_kept(gb, gl, rows, r0, keep), s_warp, &total);
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; ++k) {
        const long long r = r0 + (long long)threadIdx.x * SCAN_PER_THREAD + k;
        if (r < rows) map[r] = keep[k] ? idx++ : -1;
    }
}

// ------------------------------------------------------------------------------------ pass 3
// One CTA walks a contiguous block of joint nodes; thread i owns the 16-byte column groups i, i+256, ... of every
// row (32 columns per thread -> V <= 8192), so the column sums of dlogits (= the fc2 bias
// gradient) accumulate in registers for free.  GRAD_RU rows are in flight per thread.
// COMPACT: a row r with row_map[r] < 0 is neither read nor written; a kept row's gradient goes to row row_map[r] of dlogits (= dz_c)
// and its joint activations h[r] are copied to h_c[row_map[r]].  The CTA blocks and the column sums are those of the dense form.
constexpr int GRAD_THREADS = 256;
template <typename T> struct GradCfg { static constexpr int MAXG = 32 / Vec16<T>::N; };   // 16-byte groups per thread: V <= 8192 for bf16 and f32
// ROWY (the pruned loss): row r is not node (b, t, u = r % U1) but a gathered one; its label column is row_y[r] (-1: none).
template <typename T, int GRAD_RU, int MINB, bool COMPACT, bool ROWY = false>
__global__ void __launch_bounds__(GRAD_THREADS, MINB) rnnt_grad_kernel(const T* logits, const int* __restrict__ labels,
                                                                    const int* __restrict__ label_lens, RnntDims d,
                                                                    const float* __restrict__ lse_in, const float* __restrict__ gb_in,
                                                                    const float* __restrict__ gl_in, T* dlogits, float* __restrict__ colsum,
                                                                    long long rows_per_cta, const int* __restrict__ row_map,
                                                                    const T* __restrict__ h, T* __restrict__ h_c, int H,
                                                                    const int* __restrict__ row_y = nullptr) {
    constexpr int VN = Vec16<T>::N;
    constexpr int GRAD_MAXG = GradCfg<T>::MAXG;
    extern __shared__ float gsm[];                          // per-row scalars of this CTA's block: gb, gl, lse*log2e, label (, map)
    float* s_gb = gsm;
    float* s_gl = gsm + rows_per_cta;
    float* s_l2 = gsm + 2 * rows_per_cta;
    int* s_y = reinterpret_cast<int*>(gsm + 3 * rows_per_cta);
    int* s_map = reinterpret_cast<int*>(gsm + 4 * rows_per_cta);
    const long long rows = (long long)d.B * d.T * d.U1;
    const long long r0 = (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min(rows, r0 + rows_per_cta);
    const int nvec_ld = d.ldv / VN;
    const int tid = threadIdx.x;
    for (long long row = r0 + tid; row < r1; row += GRAD_THREADS) {
        const int i = (int)(row - r0);
        s_gb[i] = gb_in[row];
        s_gl[i] = gl_in[row];
        s_l2[i] = lse_in[row] * kLog2e;
        if (ROWY) {
            s_y[i] = row_y[row];
        } else {
            const int u = (int)(row % d.U1);
            const int b = (int)(row / ((long long)d.T * d.U1));
            s_y[i] = (u < label_lens[b]) ? labels[(size_t)b * d.ld_labels + u] : -1;
        }
        if (COMPACT) s_map[i] = row_map[row];
    }
    __syncthreads();
    const int h_vec = COMPACT ? H / 8 : 0;                  // 16-byte groups of an h row (bf16): one per thread, H <= 2048
    float cs[GRAD_MAXG][VN];
#pragma unroll
    for (int gq = 0; gq < GRAD_MAXG; ++gq)
#pragma unroll
        for (int e = 0; e < VN; ++e) cs[gq][e] = 0.f;
    for (long long rb = r0; rb < r1; rb += GRAD_RU) {
        uint4 q[GRAD_RU][GRAD_MAXG];
        uint4 hq[GRAD_RU];
#pragma unroll
        for (int k = 0; k < GRAD_RU; ++k) {
            const long long row = rb + k;
            if (row < r1 && (COMPACT ? s_map[row - r0] >= 0 : (s_gb[row - r0] != 0.f || s_gl[row - r0] != 0.f))) {
                const uint4* vp = reinterpret_cast<const uint4*>(logits + row * (long long)d.ldv);
#pragma unroll
                for (int gq = 0; gq < GRAD_MAXG; ++gq) {
                    const int i = tid + gq * GRAD_THREADS;
                    if (i < nvec_ld) q[k][gq] = ld_plain(vp + i);
                }
                if (COMPACT && tid < h_vec) hq[k] = ld_stream(reinterpret_cast<const uint4*>(h + row * (long long)H) + tid);
            }
        }
#pragma unroll
        for (int k = 0; k < GRAD_RU; ++k) {
            const long long row = rb + k;
            if (row >= r1) continue;
            const float gb = s_gb[row - r0], gl = s_gl[row - r0];
            long long orow = row;
            if (COMPACT) {
                orow = s_map[row - r0];
                if (orow < 0) continue;                 // all-zero gradient row: not stored
                if (tid < h_vec) st_stream(reinterpret_cast<uint4*>(h_c + orow * H) + tid, hq[k]);
            }
            uint4* op = reinterpret_cast<uint4*>(dlogits + orow * (long long)d.ldv);
            if (gb == 0.f && gl == 0.f) {               // padded (or zero-probability) node: zeros, nothing read
#pragma unroll
                for (int gq = 0; gq < GRAD_MAXG; ++gq) {
                    const int i = tid + gq * GRAD_THREADS;
                    if (i < nvec_ld) st_stream(op + i, make_uint4(0, 0, 0, 0));
                }
                continue;
            }
            const int y = s_y[row - r0];
            const float l2 = s_l2[row - r0];
            const float gsum = -(gb + gl);
#pragma unroll
            for (int gq = 0; gq < GRAD_MAXG; ++gq) {
                const int i = tid + gq * GRAD_THREADS;
                if (i < nvec_ld) {
                    float f[VN];
                    Vec16<T>::unpack(q[k][gq], f);
#pragma unroll
                    for (int e = 0; e < VN; ++e) f[e] = ex2_approx(fmaf(f[e], kLog2e, -l2)) * gsum;
                    const int v0 = i * VN;
                    if (v0 == 0) f[0] += gb;                                   // blank column
                    if (y >= v0 && y < v0 + VN) {                              // label column (one thread per row)
#pragma unroll
                        for (int e = 0; e < VN; ++e) if (v0 + e == y) f[e] += gl;
                    }
                    if (v0 + VN > d.V) {                                       // row padding [V, ldv)
#pragma unroll
                        for (int e = 0; e < VN; ++e) if (v0 + e >= d.V) f[e] = 0.f;
                    }
                    const uint4 packed = Vec16<T>::pack(f);
                    st_stream(op + i, packed);
                    if (colsum) {                         // sum what was actually stored (bf16-rounded in production)
                        float w[VN];
                        Vec16<T>::unpack(packed, w);
#pragma unroll
                        for (int e = 0; e < VN; ++e) cs[gq][e] += w[e];
                    }
                }
            }
        }
    }
    if (colsum) {
        // one partial row per CTA (no atomics): colsum_partials_kernel adds them in a fixed order, so the fc2 bias
        // gradient is bit-reproducible from run to run
        float* part = colsum + (size_t)blockIdx.x * d.ldv;
#pragma unroll
        for (int gq = 0; gq < GRAD_MAXG; ++gq) {
            const int i = tid + gq * GRAD_THREADS;
            if (i < nvec_ld) {
#pragma unroll
                for (int e = 0; e < VN; ++e) part[i * VN + e] = cs[gq][e];
            }
        }
    }
}

// out[c] = sum over the n_part partial rows.  Block = 32 columns x 8 row groups; every group adds its rows in index order and the
// eight group sums are combined in a fixed order, so the result is bit-reproducible.
__global__ void __launch_bounds__(256) colsum_partials_kernel(const float* __restrict__ part, int n_part, int ld, float* __restrict__ out) {
    __shared__ float sm[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx;
    float a = 0.f;
    if (c < ld) {
        const int per = (n_part + 7) / 8;
        const int i0 = ty * per, i1 = min(n_part, i0 + per);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        int i = i0;
        for (; i + 4 <= i1; i += 4) {
            a0 += part[(size_t)(i + 0) * ld + c]; a1 += part[(size_t)(i + 1) * ld + c];
            a2 += part[(size_t)(i + 2) * ld + c]; a3 += part[(size_t)(i + 3) * ld + c];
        }
        for (; i < i1; ++i) a0 += part[(size_t)i * ld + c];
        a = (a0 + a1) + (a2 + a3);
    }
    sm[ty][tx] = a;
    __syncthreads();
    if (ty == 0 && c < ld) {
        float t = sm[0][tx];
#pragma unroll
        for (int k = 1; k < 8; ++k) t += sm[k][tx];
        out[c] = t;
    }
}

// ------------------------------------------------------------------------------------ pruned loss (pk_rnnt_pruned_loss)
// Row (b, t, r) of the [B*T*R, ldv] logits is node (t, u = s_t + r); it is masked (no log-prob, zero gradient) when t >= T_b or
// u > U_b.  Pass 1: the row log-sum-exp, one warp per row (streamed) or merged from the producing GEMM's partials.
template <typename T>
__global__ void __launch_bounds__(256) pruned_row_lse_kernel(const T* __restrict__ logits, const int* __restrict__ frame_lens,
                                                             const int* __restrict__ label_lens, const int* __restrict__ bounds, int Tt,
                                                             int R, int V, int ldv, long long rows, const float2* __restrict__ parts,
                                                             int n_parts, float* __restrict__ lse_out) {
    constexpr int VN = Vec16<T>::N;
    const int lane = threadIdx.x & 31;
    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += n_warps) {
        const long long bt = row / R;
        const int r = (int)(row - bt * R), t = (int)(bt % Tt), b = (int)(bt / Tt);
        if (t >= frame_lens[b] || bounds[bt] < 0 || bounds[bt] + r > label_lens[b]) continue;     // masked row (warp-uniform)
        float lse;
        if (parts != nullptr) {
            float m = -INFINITY, sum = 0.f;
            for (int i = 0; i < n_parts; ++i) m = fmaxf(m, parts[(size_t)i * rows + row].x);
            for (int i = 0; i < n_parts; ++i) { const float2 ps = parts[(size_t)i * rows + row]; sum += ps.y * exp2f(ps.x - m); }
            lse = (m + log2f(sum)) * kLn2;
        } else {
            const T* rp = logits + row * (long long)ldv;
            float m = -INFINITY, sum = 0.f;
            const int nfull = V / VN;
            for (int i = lane; i < nfull; i += 32) {
                float f[VN];
                Vec16<T>::unpack(ld_plain(reinterpret_cast<const uint4*>(rp) + i), f);
#pragma unroll
                for (int e = 0; e < VN; ++e) {
                    const float x = f[e] * kLog2e;
                    if (x > m) { sum *= exp2f(m - x); m = x; }
                    sum += exp2f(x - m);
                }
            }
            for (int v = nfull * VN + lane; v < V; v += 32) {
                const float x = to_f32<T>(rp[v]) * kLog2e;
                if (x > m) { sum *= exp2f(m - x); m = x; }
                sum += exp2f(x - m);
            }
            const float mw = warp_max(m);
            sum = (m == -INFINITY) ? 0.f : sum * exp2f(m - mw);
            sum = warp_sum(sum);
            lse = (mw + log2f(sum)) * kLn2;
        }
        if (lane == 0) lse_out[row] = lse;
    }
}

// Pass 2: the lattice tables.  One thread per valid node (b, t, u): inside the frame's window it reads its row's blank / label logit,
// outside it is -inf (no path through it).
template <typename T>
__global__ void __launch_bounds__(256) pruned_tables_kernel(const T* __restrict__ logits, const int* __restrict__ labels,
                                                            const int* __restrict__ frame_lens, const int* __restrict__ label_lens,
                                                            const int* __restrict__ bounds, RnntDims d, int R,
                                                            const float* __restrict__ lse, float* __restrict__ lpb_skew,
                                                            float* __restrict__ lpl_skew) {
    const long long n = (long long)d.B * d.T * d.U1;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % d.U1);
        const long long bt = i / d.U1;
        const int t = (int)(bt % d.T), b = (int)(bt / d.T);
        const int Un = label_lens[b];
        if (t >= frame_lens[b] || u > Un) continue;
        const int r = u - bounds[bt];
        const size_t sk = skew_index(d, b, t, u);
        float pb = -INFINITY, pl = -INFINITY;
        if (bounds[bt] >= 0 && r >= 0 && r < R) {
            const long long row = bt * R + r;
            const T* rp = logits + row * (long long)d.ldv;
            pb = to_f32<T>(rp[0]) - lse[row];
            if (u < Un) pl = to_f32<T>(rp[labels[(size_t)b * d.ld_labels + u]]) - lse[row];
        }
        lpb_skew[sk] = pb;
        if (u < Un) lpl_skew[sk] = pl;
    }
}

// Pass 4 (after the lattice): per-row gradient coefficients for rnnt_grad_kernel<ROWY>: the occupancies of the row's node and its
// label column; masked rows get zeros (the gradient kernel writes a zero row without reading the logits).
__global__ void __launch_bounds__(256) pruned_rows_kernel(const int* __restrict__ labels, const int* __restrict__ frame_lens,
                                                          const int* __restrict__ label_lens, const int* __restrict__ bounds, RnntDims d,
                                                          int R, const float* __restrict__ gb, const float* __restrict__ gl,
                                                          float* __restrict__ gb_row, float* __restrict__ gl_row, int* __restrict__ y_row) {
    const long long rows = (long long)d.B * d.T * R;
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < rows; row += (long long)gridDim.x * blockDim.x) {
        const long long bt = row / R;
        const int r = (int)(row - bt * R), t = (int)(bt % d.T), b = (int)(bt / d.T);
        const int Un = label_lens[b], u = bounds[bt] + r;
        float vb = 0.f, vl = 0.f;
        int y = -1;
        if (t < frame_lens[b] && bounds[bt] >= 0 && u <= Un) {
            const long long node = bt * d.U1 + u;
            vb = gb[node];
            if (u < Un) { vl = gl[node]; y = labels[(size_t)b * d.ld_labels + u]; }
        }
        gb_row[row] = vb;
        gl_row[row] = vl;
        y_row[row] = y;
    }
}

}  // namespace pk

extern "C" long long pk_rnnt_loss_workspace_bytes(int B, int T, int U1) {
    const long long nd = (long long)T + U1 - 1;
    const long long skew = (long long)B * nd * U1;
    const long long nodes = (long long)B * T * U1;
    return (2 * skew + 3 * nodes) * 4 + 2 * skew * 8 + 256;
}
// gradient-kernel grid: 3 CTAs per SM x 4 waves, rows per CTA a multiple of the 2 rows each thread keeps in flight.  Shared by the
// launch and by the column-sum workspace query.
static void rnnt_grad_grid(long long rows, long long* rpc_out, int* ggrid_out) {
    const int ru = 2;
    const int gcta = pk::num_sms() * 3 * 4;
    long long rpc = (rows + gcta - 1) / gcta;
    rpc = (rpc + ru - 1) / ru * ru;
    if (rpc > 2048) rpc = 2048;                      // 16 (compacted: 20) bytes of shared memory per row
    *rpc_out = rpc; *ggrid_out = (int)((rows + rpc - 1) / rpc);
}
extern "C" long long pk_rnnt_loss_colsum_workspace_bytes(int B, int T, int U1, int ldv) {
    int ggrid; long long rpc;
    rnnt_grad_grid((long long)B * T * U1, &rpc, &ggrid);
    return (long long)ggrid * ldv * 4;
}

// lam_d = delay penalty, fe_scale = 1 + FastEmit lambda; (0, 1) launches the plain lattice
template <bool REG>
static int lattice_allow_smem() {                    // the two ping-pong diagonals exceed the default 48 KB from U+1 = 1534 on
    static bool configured = false;
    if (!configured) {
        PK_CHECK_CUDA(cudaFuncSetAttribute(pk::rnnt_lattice_kernel<REG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           2 * 2 * (pk::LAT_MAX_G * pk::LAT_MAX_CPT + 2) * (int)sizeof(pk::lat_t)));
        configured = true;
    }
    return 0;
}

static int launch_lattice(const int* frame_lens, const int* label_lens, const pk::RnntDims& d, const float* lpb, const float* lpl,
                          double* alpha, double* beta, const float* grad_scale, float* costs, float* gb, float* gl, cudaStream_t stream,
                          float lam_d = 0.f, float fe_scale = 1.f) {
    using namespace pk;
    const int U1 = d.U1;
    const int lat_smem = 2 * 2 * (U1 + 2) * 8;
    int G = ((U1 + 31) / 32) * 32;
    if (G > LAT_MAX_G) G = LAT_MAX_G;
    const int cpt = (U1 + G - 1) / G;
    PK_CHECK_ARG(cpt <= LAT_MAX_CPT, "U too large for the lattice kernel (U+1 <= 2048)");
    if (lam_d != 0.f || fe_scale != 1.f) {
        const int rc = lattice_allow_smem<true>();
        if (rc) return rc;
        rnnt_lattice_kernel<true><<<d.B, 2 * G, lat_smem, stream>>>(frame_lens, label_lens, d, G, cpt, lpb, lpl, alpha, beta, grad_scale,
                                                                    costs, gb, gl, (lat_t)lam_d, fe_scale);
    } else {
        const int rc = lattice_allow_smem<false>();
        if (rc) return rc;
        rnnt_lattice_kernel<false><<<d.B, 2 * G, lat_smem, stream>>>(frame_lens, label_lens, d, G, cpt, lpb, lpl, alpha, beta, grad_scale,
                                                                     costs, gb, gl, 0.0, 1.f);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

// pass 1: lse [nodes] and the skewed tables, merged from the producing GEMM's row partials (row_lse) or streamed from the logits
static int launch_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                         const pk::RnntDims& d, const float* row_lse, int n_parts, float* lse, float* lpb, float* lpl, cudaStream_t stream) {
    using namespace pk;
    const long long rows = (long long)d.B * d.T * d.U1;
    const int warps_per_cta = 8;
    long long want = (rows + warps_per_cta - 1) / warps_per_cta;
    const long long cap = (long long)num_sms() * 8 * 4;      // persistent grid-stride: 8 CTAs/SM x 4 waves
    const int grid = (int)(want < cap ? want : cap);
    if (row_lse != nullptr) {
        PK_CHECK_ARG(n_parts >= 1, "n_parts must be >= 1");
        const int fgrid = (int)((rows + 255) / 256 < (long long)num_sms() * 8 ? (rows + 255) / 256 : (long long)num_sms() * 8);
        if (dtype == PK_BF16)
            rnnt_rowfinish_kernel<__nv_bfloat16><<<fgrid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(logits), labels, frame_lens,
                                                                           label_lens, d, reinterpret_cast<const float2*>(row_lse), n_parts,
                                                                           lse, lpb, lpl);
        else
            rnnt_rowfinish_kernel<float><<<fgrid, 256, 0, stream>>>(reinterpret_cast<const float*>(logits), labels, frame_lens, label_lens, d,
                                                                   reinterpret_cast<const float2*>(row_lse), n_parts, lse, lpb, lpl);
    } else if (dtype == PK_BF16)
        rnnt_rowstats_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(logits), labels,
                                                                     frame_lens, label_lens, d, lse, lpb, lpl);
    else
        rnnt_rowstats_kernel<float><<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(logits), labels, frame_lens,
                                                              label_lens, d, lse, lpb, lpl);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

// FastEmit (lambda_f) and the delay penalty (lambda_d) of the *_reg entry points (DESIGN.md "FastEmit and delay penalty"); the plain
// entry points pass (0, 0), which launches the plain lattice.
static int check_emission_reg(float fastemit_lambda, float delay_penalty) {
    PK_CHECK_ARG(std::isfinite(fastemit_lambda) && fastemit_lambda >= 0.f, "fastemit_lambda must be finite and >= 0");
    PK_CHECK_ARG(std::isfinite(delay_penalty) && delay_penalty >= 0.f, "delay_penalty must be finite and >= 0");
    return 0;
}

static int rnnt_loss_impl(const void* logits, int dtype, const int* labels, const int* frame_lens,
                          const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                          const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                          long long workspace_bytes, const float* row_lse, int n_parts, int* row_map, int* row_count,
                          const void* h, int H, void* h_c, void* stream_v, float fastemit_lambda, float delay_penalty) {
    using namespace pk;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    {
        const int rc = check_emission_reg(fastemit_lambda, delay_penalty);
        if (rc) return rc;
    }
    PK_CHECK_ARG(dtype == PK_F32 || dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && V > 1, "bad dims");
    const int vn = dtype == PK_F32 ? 4 : 8;
    PK_CHECK_ARG(ldv >= V && ldv % vn == 0, "ldv must be >= V and a multiple of 16 bytes");
    PK_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "logits not 16B aligned");
    PK_CHECK_ARG(dlogits == nullptr || (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0, "dlogits not 16B aligned");
    PK_CHECK_ARG(workspace_bytes >= pk_rnnt_loss_workspace_bytes(B, T, U1), "workspace too small");
    RnntDims d{B, T, U1, V, ldv, ld_labels, T + U1 - 1};
    const size_t skew = (size_t)B * d.ND * U1, nodes = (size_t)B * T * U1;
    double* wsd = reinterpret_cast<double*>(workspace);          // doubles first (8-byte alignment)
    double* alpha = wsd; double* beta = alpha + skew;
    float* lpb = reinterpret_cast<float*>(beta + skew); float* lpl = lpb + skew;
    float* lse = lpl + skew; float* gb = lse + nodes; float* gl = gb + nodes;

    const long long rows = (long long)nodes;
    {
        const int rc = launch_tables(logits, dtype, labels, frame_lens, label_lens, d, row_lse, n_parts, lse, lpb, lpl, stream);
        if (rc) return rc;
    }
    {
        const int rc = launch_lattice(frame_lens, label_lens, d, lpb, lpl, alpha, beta, grad_scale, costs, gb, gl, stream, delay_penalty,
                                      1.f + fastemit_lambda);
        if (rc) return rc;
    }
    if (dlogits != nullptr) {
        PK_CHECK_ARG(ldv <= 8192, "V too large for the gradient kernel (V <= 8192)");
        int ggrid; long long rpc;
        rnnt_grad_grid(rows, &rpc, &ggrid);
        float* cs_part = nullptr;                        // [ggrid][ldv] per-CTA partial column sums, after the lattice workspace
        if (dlogits_colsum) {
            const long long base_bytes = pk_rnnt_loss_workspace_bytes(B, T, U1);
            PK_CHECK_ARG(workspace_bytes >= base_bytes + (long long)ggrid * ldv * 4,
                         "workspace too small for the column sums (add pk_rnnt_loss_colsum_workspace_bytes)");
            cs_part = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + base_bytes);
        }
        if (row_map != nullptr) {
            // the scan's tile counts live in the alpha / beta area of the workspace, which nothing reads after the lattice
            const int n_tiles = (int)((rows + SCAN_TILE - 1) / SCAN_TILE);
            int* tile_count = reinterpret_cast<int*>(alpha);
            grad_rows_count_kernel<<<n_tiles, SCAN_THREADS, 0, stream>>>(gb, gl, rows, tile_count);
            PK_CHECK_LAUNCH(); count_launch();
            grad_rows_scan_kernel<__nv_bfloat16><<<1, SCAN_THREADS, 0, stream>>>(tile_count, n_tiles, row_count, rows,
                                                                                 reinterpret_cast<__nv_bfloat16*>(dlogits), ldv,
                                                                                 reinterpret_cast<__nv_bfloat16*>(h_c), H);
            PK_CHECK_LAUNCH(); count_launch();
            grad_rows_map_kernel<<<n_tiles, SCAN_THREADS, 0, stream>>>(gb, gl, rows, tile_count, row_map);
            PK_CHECK_LAUNCH(); count_launch();
        }
        const size_t gsmem = (size_t)rpc * (row_map != nullptr ? 20 : 16);
#define PK_GRAD_LAUNCH(TT, RU, MB, CP)                                                                                     \
        rnnt_grad_kernel<TT, RU, MB, CP><<<ggrid, GRAD_THREADS, gsmem, stream>>>(reinterpret_cast<const TT*>(logits), labels, label_lens, d, \
                                                                                lse, gb, gl, reinterpret_cast<TT*>(dlogits), cs_part, rpc,  \
                                                                                row_map, reinterpret_cast<const TT*>(h),                    \
                                                                                reinterpret_cast<TT*>(h_c), H)
        if (row_map != nullptr) PK_GRAD_LAUNCH(__nv_bfloat16, 2, 3, true);
        else if (dtype == PK_BF16) PK_GRAD_LAUNCH(__nv_bfloat16, 2, 3, false);
        else PK_GRAD_LAUNCH(float, 2, 2, false);
#undef PK_GRAD_LAUNCH
        PK_CHECK_LAUNCH(); count_launch();
        if (dlogits_colsum) {
            colsum_partials_kernel<<<(ldv + 31) / 32, 256, 0, stream>>>(cs_part, ggrid, ldv, dlogits_colsum);
            PK_CHECK_LAUNCH(); count_launch();
        }
    }
    return 0;
}

extern "C" int pk_rnnt_loss_fwd_bwd_reg(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                        const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                        const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                                        long long workspace_bytes, float fastemit_lambda, float delay_penalty, void* stream) {
    return rnnt_loss_impl(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs, dlogits,
                          dlogits_colsum, workspace, workspace_bytes, nullptr, 0, nullptr, nullptr, nullptr, 0, nullptr, stream,
                          fastemit_lambda, delay_penalty);
}

extern "C" int pk_rnnt_loss_fwd_bwd(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                    const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                    const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                                    long long workspace_bytes, void* stream) {
    return pk_rnnt_loss_fwd_bwd_reg(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs, dlogits,
                                    dlogits_colsum, workspace, workspace_bytes, 0.f, 0.f, stream);
}

extern "C" int pk_rnnt_loss_fwd_bwd_lse_reg(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                            const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                            const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                                            long long workspace_bytes, const float* row_lse, int n_parts, float fastemit_lambda,
                                            float delay_penalty, void* stream) {
    PK_CHECK_ARG(row_lse != nullptr, "row_lse is null");
    return rnnt_loss_impl(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs, dlogits,
                          dlogits_colsum, workspace, workspace_bytes, row_lse, n_parts, nullptr, nullptr, nullptr, 0, nullptr, stream,
                          fastemit_lambda, delay_penalty);
}

extern "C" int pk_rnnt_loss_fwd_bwd_lse(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                        const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                        const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                                        long long workspace_bytes, const float* row_lse, int n_parts, void* stream) {
    return pk_rnnt_loss_fwd_bwd_lse_reg(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs,
                                        dlogits, dlogits_colsum, workspace, workspace_bytes, row_lse, n_parts, 0.f, 0.f, stream);
}

extern "C" int pk_rnnt_loss_fwd_bwd_compact_reg(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                                const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                                const float* grad_scale, float* costs, void* dz_c, float* dlogits_colsum, void* workspace,
                                                long long workspace_bytes, const float* row_lse, int n_parts, const void* h, int H,
                                                void* h_c, int* row_map, int* row_count, float fastemit_lambda, float delay_penalty,
                                                void* stream) {
    PK_CHECK_ARG(dtype == PK_BF16, "the compacted gradient is bf16 only");
    PK_CHECK_ARG(dz_c != nullptr && row_map != nullptr && row_count != nullptr && h != nullptr && h_c != nullptr, "null pointer");
    PK_CHECK_ARG(H > 0 && H % 8 == 0 && H / 8 <= pk::GRAD_THREADS, "H must be a multiple of 8, <= 2048");
    PK_CHECK_ARG(dz_c != logits, "dz_c must not alias the logits");
    PK_CHECK_ARG((reinterpret_cast<uintptr_t>(h) & 15) == 0 && (reinterpret_cast<uintptr_t>(h_c) & 15) == 0, "h / h_c not 16B aligned");
    return rnnt_loss_impl(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs, dz_c,
                          dlogits_colsum, workspace, workspace_bytes, row_lse, n_parts, row_map, row_count, h, H, h_c, stream,
                          fastemit_lambda, delay_penalty);
}

extern "C" int pk_rnnt_loss_fwd_bwd_compact(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                            const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                            const float* grad_scale, float* costs, void* dz_c, float* dlogits_colsum, void* workspace,
                                            long long workspace_bytes, const float* row_lse, int n_parts, const void* h, int H,
                                            void* h_c, int* row_map, int* row_count, void* stream) {
    return pk_rnnt_loss_fwd_bwd_compact_reg(logits, dtype, labels, frame_lens, label_lens, B, T, U1, V, ldv, ld_labels, grad_scale, costs,
                                            dz_c, dlogits_colsum, workspace, workspace_bytes, row_lse, n_parts, h, H, h_c, row_map,
                                            row_count, 0.f, 0.f, stream);
}

static long long lattice_ws_bytes(int B, int T, int U1) { return 2 * (long long)B * ((long long)T + U1 - 1) * U1 * 8; }
extern "C" int pk_rnnt_lattice_workspace(int B, int T, int U1, long long* bytes) {
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && bytes != nullptr, "bad dims or null pointer");
    *bytes = lattice_ws_bytes(B, T, U1);
    return 0;
}

extern "C" int pk_rnnt_lattice_reg(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew,
                                   const float* lpl_skew, const float* grad_scale, float* costs, float* gb, float* gl, void* workspace,
                                   long long workspace_bytes, float fastemit_lambda, float delay_penalty, void* stream) {
    using namespace pk;
    {
        const int rc = check_emission_reg(fastemit_lambda, delay_penalty);
        if (rc) return rc;
    }
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0, "bad dims");
    PK_CHECK_ARG(lpb_skew && lpl_skew && costs && gb && gl && workspace, "null pointer");
    PK_CHECK_ARG(workspace_bytes >= lattice_ws_bytes(B, T, U1), "workspace too small");
    RnntDims d{B, T, U1, 2, 2, 1, T + U1 - 1};
    const size_t skew = (size_t)B * d.ND * U1;
    double* alpha = reinterpret_cast<double*>(workspace);
    return launch_lattice(frame_lens, label_lens, d, lpb_skew, lpl_skew, alpha, alpha + skew, grad_scale, costs, gb, gl,
                          reinterpret_cast<cudaStream_t>(stream), delay_penalty, 1.f + fastemit_lambda);
}

extern "C" int pk_rnnt_lattice(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew,
                               const float* lpl_skew, const float* grad_scale, float* costs, float* gb, float* gl, void* workspace,
                               long long workspace_bytes, void* stream) {
    return pk_rnnt_lattice_reg(frame_lens, label_lens, B, T, U1, lpb_skew, lpl_skew, grad_scale, costs, gb, gl, workspace, workspace_bytes,
                               0.f, 0.f, stream);
}

// workspace of pk_rnnt_pruned_loss: alpha, beta (f64 skew), lpb, lpl (f32 skew), gb, gl (f32 nodes), lse, gb_row, gl_row, y_row
// (per pruned row), then the gradient pass's per-CTA column-sum partials
static long long pruned_ws_parts(int B, int T, int U1, int R, int ldv, long long* colsum_off) {
    const long long skew = (long long)B * ((long long)T + U1 - 1) * U1, nodes = (long long)B * T * U1, rows = (long long)B * T * R;
    const long long base = 2 * skew * 8 + 2 * skew * 4 + 2 * nodes * 4 + 4 * rows * 4;
    const long long off = (base + 255) / 256 * 256;
    int ggrid; long long rpc;
    rnnt_grad_grid(rows, &rpc, &ggrid);
    if (colsum_off) *colsum_off = off;
    return off + (long long)ggrid * ldv * 4;
}
extern "C" int pk_rnnt_pruned_loss_workspace(int B, int T, int U1, int R, int ldv, long long* bytes) {
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && R >= 1 && ldv > 0 && bytes != nullptr, "bad dims or null pointer");
    *bytes = pruned_ws_parts(B, T, U1, R, ldv, nullptr);
    return 0;
}

// the pruned loss's passes 1 and 2: the row log-sum-exp lse [B*T*R], then tables with -inf outside each frame's window
static int launch_pruned_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                                 const int* bounds, const pk::RnntDims& d, int R, const float* row_lse, int n_parts, float* lse, float* lpb,
                                 float* lpl, cudaStream_t stream) {
    using namespace pk;
    const long long rows = (long long)d.B * d.T * R;
    const int wgrid = (int)std::min<long long>((rows + 7) / 8, (long long)num_sms() * 32);
    const long long nn = (long long)d.B * d.T * d.U1;
    const int ngrid = (int)std::min<long long>((nn + 255) / 256, (long long)num_sms() * 8);
    if (dtype == PK_BF16) {
        using TT = __nv_bfloat16;
        pruned_row_lse_kernel<TT><<<wgrid, 256, 0, stream>>>((const TT*)logits, frame_lens, label_lens, bounds, d.T, R, d.V, d.ldv, rows,
                                                            (const float2*)row_lse, n_parts, lse);
        PK_CHECK_LAUNCH(); count_launch();
        pruned_tables_kernel<TT><<<ngrid, 256, 0, stream>>>((const TT*)logits, labels, frame_lens, label_lens, bounds, d, R, lse, lpb, lpl);
    } else {
        pruned_row_lse_kernel<float><<<wgrid, 256, 0, stream>>>((const float*)logits, frame_lens, label_lens, bounds, d.T, R, d.V, d.ldv,
                                                               rows, (const float2*)row_lse, n_parts, lse);
        PK_CHECK_LAUNCH(); count_launch();
        pruned_tables_kernel<float><<<ngrid, 256, 0, stream>>>((const float*)logits, labels, frame_lens, label_lens, bounds, d, R, lse, lpb,
                                                               lpl);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_pruned_loss_reg(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                                       const int* bounds, int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* grad_scale,
                                       float* costs, void* dlogits, float* dlogits_colsum, void* workspace, long long workspace_bytes,
                                       const float* row_lse, int n_parts, float fastemit_lambda, float delay_penalty, void* stream_v) {
    using namespace pk;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    {
        const int rc = check_emission_reg(fastemit_lambda, delay_penalty);
        if (rc) return rc;
    }
    PK_CHECK_ARG(dtype == PK_F32 || dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && R >= 1 && V > 1, "bad dims");
    const int vn = dtype == PK_F32 ? 4 : 8;
    PK_CHECK_ARG(ldv >= V && ldv % vn == 0, "ldv must be >= V and a multiple of 16 bytes");
    PK_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "logits not 16B aligned");
    PK_CHECK_ARG(dlogits == nullptr || (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0, "dlogits not 16B aligned");
    PK_CHECK_ARG(row_lse == nullptr || n_parts >= 1, "n_parts must be >= 1");
    PK_CHECK_ARG(dlogits == nullptr || ldv <= 8192, "V too large for the gradient kernel (V <= 8192)");
    long long cs_off;
    PK_CHECK_ARG(workspace_bytes >= pruned_ws_parts(B, T, U1, R, ldv, &cs_off), "workspace too small");
    RnntDims d{B, T, U1, V, ldv, ld_labels, T + U1 - 1};
    const size_t skew = (size_t)B * d.ND * U1, nodes = (size_t)B * T * U1;
    const long long rows = (long long)B * T * R;
    double* alpha = reinterpret_cast<double*>(workspace); double* beta = alpha + skew;
    float* lpb = reinterpret_cast<float*>(beta + skew); float* lpl = lpb + skew;
    float* gb = lpl + skew; float* gl = gb + nodes;
    float* lse = gl + nodes; float* gb_row = lse + rows; float* gl_row = gb_row + rows;
    int* y_row = reinterpret_cast<int*>(gl_row + rows);
    {
        const int rc = launch_pruned_tables(logits, dtype, labels, frame_lens, label_lens, bounds, d, R, row_lse, n_parts, lse, lpb, lpl,
                                            stream);
        if (rc) return rc;
    }
    {
        const int rc = launch_lattice(frame_lens, label_lens, d, lpb, lpl, alpha, beta, grad_scale, costs, gb, gl, stream, delay_penalty,
                                      1.f + fastemit_lambda);
        if (rc) return rc;
    }
    if (dlogits == nullptr) return 0;
    const int rgrid = (int)std::min<long long>((rows + 255) / 256, (long long)num_sms() * 8);
    pruned_rows_kernel<<<rgrid, 256, 0, stream>>>(labels, frame_lens, label_lens, bounds, d, R, gb, gl, gb_row, gl_row, y_row);
    PK_CHECK_LAUNCH(); count_launch();
    int ggrid; long long rpc;
    rnnt_grad_grid(rows, &rpc, &ggrid);
    float* cs_part = dlogits_colsum ? reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + cs_off) : nullptr;
    RnntDims dr{B, T, R, V, ldv, ld_labels, 0};          // the gradient kernel's rows are the B*T*R pruned rows
    const size_t gsmem = (size_t)rpc * 16;
    if (dtype == PK_BF16)
        rnnt_grad_kernel<__nv_bfloat16, 2, 3, false, true><<<ggrid, GRAD_THREADS, gsmem, stream>>>(
            (const __nv_bfloat16*)logits, labels, label_lens, dr, lse, gb_row, gl_row, (__nv_bfloat16*)dlogits, cs_part, rpc, nullptr,
            nullptr, nullptr, 0, y_row);
    else
        rnnt_grad_kernel<float, 2, 2, false, true><<<ggrid, GRAD_THREADS, gsmem, stream>>>(
            (const float*)logits, labels, label_lens, dr, lse, gb_row, gl_row, (float*)dlogits, cs_part, rpc, nullptr, nullptr, nullptr, 0,
            y_row);
    PK_CHECK_LAUNCH(); count_launch();
    if (dlogits_colsum) {
        colsum_partials_kernel<<<(ldv + 31) / 32, 256, 0, stream>>>(cs_part, ggrid, ldv, dlogits_colsum);
        PK_CHECK_LAUNCH(); count_launch();
    }
    return 0;
}

extern "C" int pk_rnnt_pruned_loss(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                                   const int* bounds, int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* grad_scale,
                                   float* costs, void* dlogits, float* dlogits_colsum, void* workspace, long long workspace_bytes,
                                   const float* row_lse, int n_parts, void* stream) {
    return pk_rnnt_pruned_loss_reg(logits, dtype, labels, frame_lens, label_lens, bounds, B, T, U1, R, V, ldv, ld_labels, grad_scale, costs,
                                   dlogits, dlogits_colsum, workspace, workspace_bytes, row_lse, n_parts, 0.f, 0.f, stream);
}

// ------------------------------------------------------------------------------------ forced alignment entry points
static int check_logits_args(const void* logits, int dtype, int B, int T, int U1, int V, int ldv) {
    PK_CHECK_ARG(dtype == PK_F32 || dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && V > 1, "bad dims");
    const int vn = dtype == PK_F32 ? 4 : 8;
    PK_CHECK_ARG(ldv >= V && ldv % vn == 0, "ldv must be >= V and a multiple of 16 bytes");
    PK_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "logits not 16B aligned");
    return 0;
}

extern "C" int pk_rnnt_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, int B, int T,
                              int U1, int V, int ldv, int ld_labels, const float* row_lse, int n_parts, float* lse, float* lpb_skew,
                              float* lpl_skew, void* stream) {
    const int rc = check_logits_args(logits, dtype, B, T, U1, V, ldv);
    if (rc) return rc;
    PK_CHECK_ARG(lse && lpb_skew && lpl_skew, "null pointer");
    pk::RnntDims d{B, T, U1, V, ldv, ld_labels, T + U1 - 1};
    return launch_tables(logits, dtype, labels, frame_lens, label_lens, d, row_lse, n_parts, lse, lpb_skew, lpl_skew,
                         reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int pk_rnnt_pruned_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                                     const int* bounds, int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* row_lse,
                                     int n_parts, float* lse, float* lpb_skew, float* lpl_skew, void* stream) {
    const int rc = check_logits_args(logits, dtype, B, T, U1, V, ldv);
    if (rc) return rc;
    PK_CHECK_ARG(R >= 1, "R must be >= 1");
    PK_CHECK_ARG(row_lse == nullptr || n_parts >= 1, "n_parts must be >= 1");
    PK_CHECK_ARG(bounds && lse && lpb_skew && lpl_skew, "null pointer");
    pk::RnntDims d{B, T, U1, V, ldv, ld_labels, T + U1 - 1};
    return launch_pruned_tables(logits, dtype, labels, frame_lens, label_lens, bounds, d, R, row_lse, n_parts, lse, lpb_skew, lpl_skew,
                                reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int pk_rnnt_lattice_costs(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew,
                                     const float* lpl_skew, float* costs, void* workspace, long long workspace_bytes, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0, "bad dims");
    PK_CHECK_ARG(lpb_skew && lpl_skew && costs && workspace, "null pointer");
    PK_CHECK_ARG(workspace_bytes >= lattice_ws_bytes(B, T, U1), "workspace too small");
    RnntDims d{B, T, U1, 2, 2, 1, T + U1 - 1};
    const size_t skew = (size_t)B * d.ND * U1;
    double* alpha = reinterpret_cast<double*>(workspace);
    return launch_lattice(frame_lens, label_lens, d, lpb_skew, lpl_skew, alpha, alpha + skew, nullptr, costs, nullptr, nullptr,
                          reinterpret_cast<cudaStream_t>(stream));
}

static long long viterbi_ws_bytes(int B, int T, int U1) { return (long long)B * ((long long)T + U1 - 1) * ((U1 + 31) / 32) * 4; }
extern "C" int pk_rnnt_viterbi_workspace(int B, int T, int U1, long long* bytes) {
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && bytes != nullptr, "bad dims or null pointer");
    *bytes = viterbi_ws_bytes(B, T, U1);
    return 0;
}

extern "C" int pk_rnnt_viterbi(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew,
                               const float* lpl_skew, float* score, int* emit_frames, int ld_emit, void* workspace, long long workspace_bytes,
                               void* stream) {
    using namespace pk;
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && ld_emit >= 0, "bad dims");
    PK_CHECK_ARG(lpb_skew && lpl_skew && score && workspace && (emit_frames || ld_emit == 0), "null pointer");
    PK_CHECK_ARG(ld_emit >= U1 - 1, "ld_emit must be >= U1 - 1");
    PK_CHECK_ARG(workspace_bytes >= viterbi_ws_bytes(B, T, U1), "workspace too small");
    int G = ((U1 + 31) / 32) * 32;
    if (G > LAT_MAX_G) G = LAT_MAX_G;
    const int cpt = (U1 + G - 1) / G;
    PK_CHECK_ARG(cpt <= LAT_MAX_CPT, "U too large for the Viterbi kernel (U+1 <= 2048)");
    RnntDims d{B, T, U1, 2, 2, 1, T + U1 - 1};
    const int smem = 2 * (U1 + 2) * (int)sizeof(lat_t);           // <= 32.8 KB: no opt-in needed
    rnnt_viterbi_kernel<<<B, G, smem, reinterpret_cast<cudaStream_t>(stream)>>>(frame_lens, label_lens, d, G, cpt, lpb_skew, lpl_skew,
                                                                                reinterpret_cast<unsigned*>(workspace), score, emit_frames,
                                                                                ld_emit);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
