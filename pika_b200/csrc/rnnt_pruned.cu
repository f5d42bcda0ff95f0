// Pruned RNN-T loss (Kuang et al., 2022): the simple joiner's loss, the pruning bounds and the pruned gated joint.
//
//   simple joiner    z[t,u] = am[t] + lm[u] (two linear projections of the encoder / prediction-net outputs).  Its normaliser
//                    N[t,u] = log(E_t . P_u) + max(am_t) + max(lm_u), E = exp(am - rowmax), P = exp(lm - rowmax), is one batched
//                    [T x V].[V x U1] GEMM (pk_gemm_bf16) instead of a [T, U1, V] tensor:
//     pk_rnnt_simple_prep    row max and exp of am / lm -> the bf16 (hi[, lo]) GEMM operands E, P, zero pad columns and rows
//     pk_rnnt_simple_tables  S = E.P^T, the maxes and the blank / label gathers -> lpb, lpl in the lattice's skewed layout
//                            (then pk_rnnt_lattice, rnnt_loss.cu, gives the costs and the occupancies gb, gl)
//     pk_rnnt_simple_w       W = scale * gamma / S, gamma = -(gb + gl): the operand of the two gradient GEMMs W.P and W^T.E
//     pk_rnnt_simple_grad    dam = E (.) (W P) + blank / label terms, dlm = P (.) (W^T E) + blank / label terms; one CTA per row,
//                            the terms added by one thread in a fixed order (no atomics)
//     pk_rnnt_simple_smooth_stats, _tables_smooth, _grad_smooth   the same with LM-only / AM-only log-probs mixed into the lattice
//   pk_rnnt_prune_bounds     the simple occupancies -> the first label position s[b, t] of each frame's window of R positions
//   pk_joint_gate_pruned_fwd / _bwd   the factored gate h = tanh(ex1 + py1) * sigmoid(exg + pyg) on the B*T*R rows (t, s_t + r)
// The pruned loss itself (tables from the [B*T*R, ldv] logits, lattice, gradient) is pk_rnnt_pruned_loss in rnnt_loss.cu, next to
// the lattice and gradient kernels it reuses.
#include <cfloat>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

// S = E_t . P_u underflows when the two rows' large entries do not overlap; it is clamped to 2^-100 before the log, so
// N >= max(am_t) + max(lm_u) - 100 ln 2 and every log-prob stays finite.  A clamped node's normaliser is a constant in the gradient.
constexpr float kSimpleFloor = 7.8886090522101181e-31f;   // 2^-100

PK_DEVICE float block_reduce_max(float v, float* s_red) {   // blockDim.x == 256
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = s_red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) r = fmaxf(r, s_red[i]);
    __syncthreads();
    return r;
}

// one CTA per output row (b, i), i < n_out: rows i < n_in hold exp(src - rowmax) over the V columns, zeros in [V, ld_out);
// rows i >= n_in (the padding of the batched GEMM's N / K extent) are all zero
__global__ void __launch_bounds__(256) simple_prep_kernel(const float* __restrict__ src, int ld_src, int V, int n_in, int n_out,
                                                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_out,
                                                          float* __restrict__ rmax) {
    __shared__ float s_red[8];
    const int b = blockIdx.x / n_out, i = blockIdx.x - b * n_out;
    __nv_bfloat16* h = hi + (long long)blockIdx.x * ld_out;
    __nv_bfloat16* l = lo ? lo + (long long)blockIdx.x * ld_out : nullptr;
    if (i >= n_in) {
        for (int c = threadIdx.x; c < ld_out; c += 256) {
            h[c] = __float2bfloat16_rn(0.f);
            if (l) l[c] = __float2bfloat16_rn(0.f);
        }
        return;
    }
    const long long srow = (long long)b * n_in + i;
    const float* x = src + srow * ld_src;
    float m = -INFINITY;
    for (int c = threadIdx.x; c < V; c += 256) m = fmaxf(m, x[c]);
    m = block_reduce_max(m, s_red);
    if (threadIdx.x == 0) rmax[srow] = m;
    for (int c = threadIdx.x; c < ld_out; c += 256) {
        const float e = c < V ? expf(x[c] - m) : 0.f;
        const __nv_bfloat16 eh = __float2bfloat16_rn(e);
        h[c] = eh;
        if (l) l[c] = __float2bfloat16_rn(e - __bfloat162float(eh));
    }
}

PK_DEVICE size_t skew_at(int ND, int U1, int b, int t, int u) { return ((size_t)b * ND + (t + u)) * U1 + u; }

PK_DEVICE float block_reduce_sum(float v, float* s_red) {   // blockDim.x == 256; the partials are added in warp order
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = s_red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) r += s_red[i];
    __syncthreads();
    return r;
}

// ------------------------------------------------------------------------------------ smoothing statistics
// The LM-only / AM-only terms' normalisers and the batch unigram q (DESIGN.md "Pruned RNN-T").  Rows outside the valid lengths are
// written 0 and never read; they enter no sum.
constexpr int kSmoothRowChunk = 64;            // lm rows per column-partial CTA of the unigram

// one CTA per row i < n_rows of utterance b (rows with i > last valid are written 0):
//   out = rmax + log sum_{v<V} exp(src + (lq ? lq : 0) - rmax).  With lq = log q <= 0, rmax (the row max of src) still bounds the
//   exponents, and the term at the row's argmax is >= q_min = 1e-10, so the sum cannot underflow to 0.
__global__ void __launch_bounds__(256) smooth_lse_kernel(const float* __restrict__ src, int ldv, int V, const float* __restrict__ rmax,
                                                         const float* __restrict__ lq, const int* __restrict__ lens, int len_off,
                                                         int n_rows, float* __restrict__ out) {
    __shared__ float s_red[8];
    const int b = blockIdx.x / n_rows, i = blockIdx.x - b * n_rows;
    if (i >= lens[b] + len_off) {
        if (threadIdx.x == 0) out[blockIdx.x] = 0.f;
        return;
    }
    const float* x = src + (long long)blockIdx.x * ldv;
    const float m = rmax[blockIdx.x];
    float s = 0.f;
    for (int c = threadIdx.x; c < V; c += 256) s += expf(x[c] + (lq ? lq[c] : 0.f) - m);
    s = block_reduce_sum(s, s_red);
    if (threadIdx.x == 0) out[blockIdx.x] = m + logf(s);
}

// grid (ceil(ldv / 256), n_chunks): column partials part[chunk][c] = sum over the valid rows of chunk (rows chunk*64 .. +63 of the
// flattened [B*U1] lm, ascending) of exp(lm - Nl); columns >= V are 0
__global__ void __launch_bounds__(256) smooth_q_part_kernel(const float* __restrict__ lm, int ldv, int V, const float* __restrict__ Nl,
                                                            const int* __restrict__ label_lens, int B, int U1, float* __restrict__ part) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= ldv) return;
    const long long r0 = (long long)blockIdx.y * kSmoothRowChunk, n = (long long)B * U1;
    float s = 0.f;
    if (c < V) {
        for (long long r = r0; r < r0 + kSmoothRowChunk && r < n; ++r) {
            const int b = (int)(r / U1), u = (int)(r - (long long)b * U1);
            if (u <= label_lens[b]) s += expf(lm[r * ldv + c] - Nl[r]);
        }
    }
    part[(long long)blockIdx.y * ldv + c] = s;
}

// log q[c] = log(sum of the chunk partials in chunk order / sum_b (U_b + 1) + 1e-10) for c < V; 0 on the padding columns
__global__ void __launch_bounds__(256) smooth_q_finish_kernel(const float* __restrict__ part, int n_chunks, int ldv, int V,
                                                              const int* __restrict__ label_lens, int B, float* __restrict__ logq) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= ldv) return;
    if (c >= V) { logq[c] = 0.f; return; }
    long long rows = 0;
    for (int b = 0; b < B; ++b) rows += label_lens[b] + 1;
    float s = 0.f;
    for (int k = 0; k < n_chunks; ++k) s += part[(long long)k * ldv + c];
    logq[c] = logf(s / (float)rows + 1e-10f);
}

// one thread per node (b, t, u) of the valid lattice: N = log(max(S, floor)) + the two maxes; lpb = z[0] - N, lpl = z[y_{u+1}] - N.
// SMOOTH: lp = mu (z[k] - N) + lam_l (lm[u,k] - Nl[u]) + lam_a (am[t,k] + log q[k] - Na[t]), mu = 1 - lam_l - lam_a.
template <bool SMOOTH>
__global__ void __launch_bounds__(256) simple_tables_kernel(const float* __restrict__ am, const float* __restrict__ lm, int ldv,
                                                            const float* __restrict__ am_max, const float* __restrict__ lm_max,
                                                            const float* __restrict__ S, int ld_s, const int* __restrict__ labels,
                                                            int ld_labels, const int* __restrict__ frame_lens,
                                                            const int* __restrict__ label_lens, int B, int T, int U1,
                                                            float* __restrict__ lpb_skew, float* __restrict__ lpl_skew,
                                                            const float* __restrict__ Nl = nullptr, const float* __restrict__ logq = nullptr,
                                                            const float* __restrict__ Na = nullptr, float mu = 1.f, float lam_l = 0.f,
                                                            float lam_a = 0.f) {
    const long long n = (long long)B * T * U1;
    const int ND = T + U1 - 1;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % U1);
        const long long bt = i / U1;
        const int t = (int)(bt % T), b = (int)(bt / T);
        const int Tn = frame_lens[b], Un = label_lens[b];
        if (t >= Tn || u > Un) continue;
        const long long ar = bt, lr = (long long)b * U1 + u;
        const float N = logf(fmaxf(S[bt * ld_s + u], kSimpleFloor)) + am_max[ar] + lm_max[lr];
        const size_t sk = skew_at(ND, U1, b, t, u);
        if constexpr (SMOOTH) {
            const float nl = Nl[lr], na = Na[ar];
            lpb_skew[sk] = mu * ((am[ar * ldv] + lm[lr * ldv]) - N) + lam_l * (lm[lr * ldv] - nl) + lam_a * ((am[ar * ldv] + logq[0]) - na);
            if (u < Un) {
                const int y = labels[(size_t)b * ld_labels + u];
                lpl_skew[sk] = mu * ((am[ar * ldv + y] + lm[lr * ldv + y]) - N) + lam_l * (lm[lr * ldv + y] - nl) +
                               lam_a * ((am[ar * ldv + y] + logq[y]) - na);
            }
        } else {
            lpb_skew[sk] = (am[ar * ldv] + lm[lr * ldv]) - N;
            if (u < Un) {
                const int y = labels[(size_t)b * ld_labels + u];
                lpl_skew[sk] = (am[ar * ldv + y] + lm[lr * ldv + y]) - N;
            }
        }
    }
}

// W[b, t, u] = scale[b] * gamma / S for the valid, unclamped nodes, else 0 (also the columns [U1, ld_w)); bf16 hi [+ lo]
__global__ void __launch_bounds__(256) simple_w_kernel(const float* __restrict__ gb, const float* __restrict__ gl,
                                                       const float* __restrict__ S, int ld_s, const int* __restrict__ frame_lens,
                                                       const int* __restrict__ label_lens, const float* __restrict__ scale, int B,
                                                       int T, int U1, __nv_bfloat16* __restrict__ w_hi, __nv_bfloat16* __restrict__ w_lo,
                                                       int ld_w) {
    const long long n = (long long)B * T * ld_w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % ld_w);
        const long long bt = i / ld_w;
        const int t = (int)(bt % T), b = (int)(bt / T);
        float w = 0.f;
        if (u < U1 && t < frame_lens[b] && u <= label_lens[b]) {
            const float s = S[bt * ld_s + u];
            const long long node = bt * U1 + u;
            const float g = -(gb[node] + gl[node]);
            if (s >= kSimpleFloor && g != 0.f) w = (scale ? scale[b] : 1.f) * g / s;
        }
        const __nv_bfloat16 h = __float2bfloat16_rn(w);
        w_hi[i] = h;
        if (w_lo) w_lo[i] = __float2bfloat16_rn(w - __bfloat162float(h));
    }
}

// d[row] = exp(src[row] - rmax[row]) (.) G[row] over the V columns, then the blank term at column 0 and the label terms at their
// columns, each summed by one thread in a fixed order.  axis 0: rows (b, t), the terms sum over u of node (t, u); axis 1: rows (b, u),
// the terms sum over t.  G row of (b, i) is b * n_g + i.  One CTA per row, the row staged in shared memory (ldv floats).
// SMOOTH: the blank / label terms are weighted by (mu + lam), and the row gains scale * lam * Gamma * exp(src + lq - lse) with
// Gamma = -(sum of the blank terms + sum of the label terms) accumulated by the same thread in the same order (lq: log q on axis 0,
// NULL on axis 1; lse: Na or Nl).
template <typename TO, bool SMOOTH>
__global__ void __launch_bounds__(256) simple_grad_kernel(const float* __restrict__ src, int ldv, int V, const float* __restrict__ rmax,
                                                          const float* __restrict__ G, int ld_g, int n_g, int axis,
                                                          const float* __restrict__ gb, const float* __restrict__ gl,
                                                          const int* __restrict__ labels, int ld_labels, const int* __restrict__ frame_lens,
                                                          const int* __restrict__ label_lens, const float* __restrict__ scale, int T,
                                                          int U1, TO* __restrict__ out, const float* __restrict__ lq = nullptr,
                                                          const float* __restrict__ lse = nullptr, float mu = 1.f, float lam = 0.f) {
    extern __shared__ float s_row[];
    __shared__ float s_gam;
    const int n_rows_b = axis == 0 ? T : U1;
    const int b = blockIdx.x / n_rows_b, i = blockIdx.x - b * n_rows_b;
    const long long row = blockIdx.x;
    const float m = rmax[row];
    const float* x = src + row * ldv;
    const float* g = G + ((long long)b * n_g + i) * ld_g;
    for (int c = threadIdx.x; c < ldv; c += 256) s_row[c] = c < V ? expf(x[c] - m) * g[c] : 0.f;
    __syncthreads();
    if (threadIdx.x == 0) {
        const int Tn = frame_lens[b], Un = label_lens[b];
        const float sc = scale ? scale[b] : 1.f;
        const long long node0 = (long long)b * T * U1;
        if constexpr (SMOOTH) {
            const float k = sc * (mu + lam);
            float blank = 0.f, lab = 0.f;
            if (axis == 0 && i < Tn) {
                for (int u = 0; u <= Un; ++u) blank += gb[node0 + (long long)i * U1 + u];
                s_row[0] += k * blank;
                for (int u = 0; u < Un; ++u) {
                    const float g = gl[node0 + (long long)i * U1 + u];
                    lab += g;
                    s_row[labels[(size_t)b * ld_labels + u]] += k * g;
                }
            } else if (axis == 1 && i <= Un) {
                for (int t = 0; t < Tn; ++t) {
                    blank += gb[node0 + (long long)t * U1 + i];
                    lab += gl[node0 + (long long)t * U1 + i];
                }
                if (i == Un) lab = 0.f;
                s_row[0] += k * blank;
                if (i < Un) s_row[labels[(size_t)b * ld_labels + i]] += k * lab;
            }
            s_gam = -(blank + lab) * sc * lam;
        } else if (axis == 0 && i < Tn) {
            float blank = 0.f;
            for (int u = 0; u <= Un; ++u) blank += gb[node0 + (long long)i * U1 + u];
            s_row[0] += sc * blank;
            for (int u = 0; u < Un; ++u) s_row[labels[(size_t)b * ld_labels + u]] += sc * gl[node0 + (long long)i * U1 + u];
        } else if (axis == 1 && i <= Un) {
            float blank = 0.f, lab = 0.f;
            for (int t = 0; t < Tn; ++t) {
                blank += gb[node0 + (long long)t * U1 + i];
                lab += gl[node0 + (long long)t * U1 + i];
            }
            s_row[0] += sc * blank;
            if (i < Un) s_row[labels[(size_t)b * ld_labels + i]] += sc * lab;
        }
    }
    __syncthreads();
    TO* o = out + row * ldv;
    if constexpr (SMOOTH) {
        const float w = s_gam;                   // 0 on padded rows, whose lse is not defined
        if (w != 0.f) {
            const float l = lse[row];
            for (int c = threadIdx.x; c < ldv; c += 256)
                o[c] = from_f32<TO>(c < V ? s_row[c] + w * expf(x[c] + (lq ? lq[c] : 0.f) - l) : 0.f);
            return;
        }
    }
    for (int c = threadIdx.x; c < ldv; c += 256) o[c] = from_f32<TO>(s_row[c]);
}

// ------------------------------------------------------------------------------------ pruning bounds
// One CTA per utterance.  gamma(t, u) = -(ga + gb) in f32; the window sums c(t, s) = sum_{u=s}^{min(s+R-1, U)} gamma(t, u) are
// formed in double in ascending u, so the argmax (smallest s on a tie) is a function of the f32 occupancies alone.  Then the clamp
// to [L_t, H_t], the running max over t and the reverse pass s_t = max(s_t, s_{t+1} - (R-1)) (a single thread: O(T) integer work).
// Padded frames copy s_{T-1}.  An utterance with U > T (R-1) (no complete path fits in the windows) gets -1 everywhere.
__global__ void __launch_bounds__(256) prune_bounds_kernel(const float* __restrict__ ga, const float* __restrict__ gb,
                                                           const int* __restrict__ frame_lens, const int* __restrict__ label_lens,
                                                           int T, int U1, int R, int* __restrict__ bounds) {
    extern __shared__ int s_s[];
    const int b = blockIdx.x;
    const int Tn = frame_lens[b], Un = label_lens[b];
    int* out = bounds + (long long)b * T;
    const bool feasible = Tn >= 1 && Tn <= T && Un >= 0 && Un < U1 && (long long)Un <= (long long)Tn * (R - 1);
    if (!feasible) {
        for (int t = threadIdx.x; t < T; t += blockDim.x) out[t] = -1;
        return;
    }
    const int S = max(Un - R + 1, 0);
    for (int t = threadIdx.x; t < Tn; t += blockDim.x) {
        const long long node = ((long long)b * T + t) * U1;
        int best = 0;
        double best_c = -1.0;
        for (int s = 0; s <= S; ++s) {
            double c = 0.0;
            const int hi = min(s + R - 1, Un);
            for (int u = s; u <= hi; ++u) c = __dadd_rn(c, (double)(-(ga[node + u] + (gb ? gb[node + u] : 0.f))));
            if (c > best_c) { best_c = c; best = s; }
        }
        const long long lo_t = (long long)Un - R + 1 - (long long)(Tn - 1 - t) * (R - 1);
        const int L = (int)(lo_t > 0 ? lo_t : 0);
        const int H = (int)min((long long)t * (R - 1), (long long)S);
        s_s[t] = min(max(best, L), H);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < Tn; ++t) s_s[t] = max(s_s[t], s_s[t - 1]);
        for (int t = Tn - 2; t >= 0; --t) s_s[t] = max(s_s[t], s_s[t + 1] - (R - 1));
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) out[t] = s_s[t < Tn ? t : Tn - 1];
}

// ------------------------------------------------------------------------------------ pruned gated joint
// row (b, t, r) of h [B*T*R, H] is the gate at (t, u = s_t + r), u clamped to [0, U1 - 1] (rows past U are masked by the loss)
PK_DEVICE int pruned_u(int s, int r, int U1) { return min(max(s, 0) + r, U1 - 1); }

template <typename T>
__global__ void __launch_bounds__(128) gate_pruned_fwd_kernel(const T* __restrict__ ex, const T* __restrict__ py, const int* __restrict__ bounds,
                                                              T* __restrict__ h, int Tt, int U1, int R, int H) {
    const int bt = blockIdx.x, b = bt / Tt;
    const int s = bounds[bt];
    const T* e = ex + (long long)bt * 2 * H;
    for (int r = 0; r < R; ++r) {
        const T* p = py + ((long long)b * U1 + pruned_u(s, r, U1)) * 2 * H;
        T* o = h + ((long long)bt * R + r) * H;
        for (int c = threadIdx.x; c < H; c += 128) {
            const float a = jt_tanh<T>(to_f32<T>(e[c]) + to_f32<T>(p[c]));
            const float g = jt_sigmoid<T>(to_f32<T>(e[H + c]) + to_f32<T>(p[H + c]));
            o[c] = from_f32<T>(a * g);
        }
    }
}

// dex[b, t] = sum over r = 0..R-1 in order; d1 = dh g (1 - a^2), dg = dh a g (1 - g)
template <typename T>
__global__ void __launch_bounds__(128) gate_pruned_bwd_ex_kernel(const T* __restrict__ ex, const T* __restrict__ py,
                                                                 const int* __restrict__ bounds, const T* __restrict__ dh,
                                                                 T* __restrict__ dex, int Tt, int U1, int R, int H) {
    const int bt = blockIdx.x, b = bt / Tt;
    const int s = bounds[bt];
    const T* e = ex + (long long)bt * 2 * H;
    for (int c = threadIdx.x; c < H; c += 128) {
        const float e1 = to_f32<T>(e[c]), eg = to_f32<T>(e[H + c]);
        float a1 = 0.f, ag = 0.f;
        for (int r = 0; r < R; ++r) {
            const T* p = py + ((long long)b * U1 + pruned_u(s, r, U1)) * 2 * H;
            const float d = to_f32<T>(dh[((long long)bt * R + r) * H + c]);
            const float a = jt_tanh<T>(e1 + to_f32<T>(p[c])), g = jt_sigmoid<T>(eg + to_f32<T>(p[H + c]));
            a1 += d * g * (1.f - a * a);
            ag += d * a * g * (1.f - g);
        }
        dex[(long long)bt * 2 * H + c] = from_f32<T>(a1);
        dex[(long long)bt * 2 * H + H + c] = from_f32<T>(ag);
    }
}

// dpy[b, u] = sum over the frames whose window holds u, in frame order.  s is non-decreasing in t, so they are one range
// [t_lo, t_hi]: t_lo = first t with s_t + R - 1 >= u, t_hi = last t with s_t <= u.  Rows whose u was clamped carry a zero
// gradient (masked by the loss) and are not visited.
template <typename T>
__global__ void __launch_bounds__(128) gate_pruned_bwd_py_kernel(const T* __restrict__ ex, const T* __restrict__ py,
                                                                 const int* __restrict__ bounds, const T* __restrict__ dh,
                                                                 T* __restrict__ dpy, int Tt, int U1, int R, int H) {
    const int bu = blockIdx.x, b = bu / U1, u = bu - b * U1;
    const int* sb = bounds + (long long)b * Tt;
    int lo = 0, hi = Tt;                       // first t with max(s_t, 0) + R - 1 >= u
    while (lo < hi) { const int m = (lo + hi) >> 1; if (max(sb[m], 0) + R - 1 >= u) hi = m; else lo = m + 1; }
    const int t_lo = lo;
    lo = 0; hi = Tt;                           // first t with max(s_t, 0) > u
    while (lo < hi) { const int m = (lo + hi) >> 1; if (max(sb[m], 0) > u) hi = m; else lo = m + 1; }
    const int t_end = lo;
    const T* p = py + (long long)bu * 2 * H;
    for (int c = threadIdx.x; c < H; c += 128) {
        const float p1 = to_f32<T>(p[c]), pg = to_f32<T>(p[H + c]);
        float a1 = 0.f, ag = 0.f;
        for (int t = t_lo; t < t_end; ++t) {
            const long long bt = (long long)b * Tt + t;
            const int r = u - max(sb[t], 0);
            const float d = to_f32<T>(dh[(bt * R + r) * H + c]);
            const float a = jt_tanh<T>(to_f32<T>(ex[bt * 2 * H + c]) + p1), g = jt_sigmoid<T>(to_f32<T>(ex[bt * 2 * H + H + c]) + pg);
            a1 += d * g * (1.f - a * a);
            ag += d * a * g * (1.f - g);
        }
        dpy[(long long)bu * 2 * H + c] = from_f32<T>(a1);
        dpy[(long long)bu * 2 * H + H + c] = from_f32<T>(ag);
    }
}

static int grid_of(long long n) {
    const long long want = (n + 255) / 256, cap = (long long)num_sms() * 8;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace pk

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int pk_rnnt_simple_prep(const float* src, int ld_src, int V, int nb, int n_in, int n_out, void* hi, void* lo, int ld_out,
                                   float* rmax, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(src && hi && rmax, "null pointer");
    PK_CHECK_ARG(V > 0 && ld_src >= V && ld_out >= V && ld_out % 8 == 0, "need V <= ld_src, V <= ld_out, ld_out % 8 == 0");
    PK_CHECK_ARG(nb > 0 && n_in > 0 && n_out >= n_in, "bad row counts");
    simple_prep_kernel<<<nb * n_out, 256, 0, STREAM(stream)>>>(src, ld_src, V, n_in, n_out, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo,
                                                                ld_out, rmax);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_simple_tables(const float* am, const float* lm, int ldv, const float* am_max, const float* lm_max, const float* S,
                                     int ld_s, const int* labels, int ld_labels, const int* frame_lens, const int* label_lens, int B, int T,
                                     int U1, float* lpb_skew, float* lpl_skew, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && ld_s >= U1, "bad dims");
    const long long n = (long long)B * T * U1;
    simple_tables_kernel<false><<<grid_of(n), 256, 0, STREAM(stream)>>>(am, lm, ldv, am_max, lm_max, S, ld_s, labels, ld_labels, frame_lens,
                                                                         label_lens, B, T, U1, lpb_skew, lpl_skew);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

static bool smooth_scales_ok(float lam_l, float lam_a) {
    return lam_l >= 0.f && lam_a >= 0.f && (double)lam_l + (double)lam_a < 1.0;   // false for NaN too
}

extern "C" int pk_rnnt_simple_smooth_stats_workspace(int B, int U1, int ldv, long long* bytes) {
    PK_CHECK_ARG(bytes, "null pointer");
    PK_CHECK_ARG(B > 0 && U1 > 0 && ldv > 0, "bad dims");
    const long long chunks = ((long long)B * U1 + pk::kSmoothRowChunk - 1) / pk::kSmoothRowChunk;
    *bytes = chunks * ldv * 4;
    return 0;
}

extern "C" int pk_rnnt_simple_smooth_stats(const float* am, const float* lm, int ldv, int V, const float* am_max, const float* lm_max,
                                           const int* frame_lens, const int* label_lens, int B, int T, int U1, float* Nl, float* logq,
                                           float* Na, void* workspace, long long workspace_bytes, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(am && lm && am_max && lm_max && frame_lens && label_lens && Nl && logq && Na && workspace, "null pointer");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && V > 0 && ldv >= V, "bad dims");
    const int chunks = (int)(((long long)B * U1 + kSmoothRowChunk - 1) / kSmoothRowChunk);
    PK_CHECK_ARG(chunks <= 65535, "B * U1 too large for the unigram's row chunks (B * U1 <= 4194240)");
    PK_CHECK_ARG(workspace_bytes >= (long long)chunks * ldv * 4, "workspace too small (pk_rnnt_simple_smooth_stats_workspace)");
    float* part = (float*)workspace;
    const int col_blocks = (ldv + 255) / 256;
    smooth_lse_kernel<<<B * U1, 256, 0, STREAM(stream)>>>(lm, ldv, V, lm_max, nullptr, label_lens, 1, U1, Nl);
    PK_CHECK_LAUNCH(); count_launch();
    smooth_q_part_kernel<<<dim3(col_blocks, chunks), 256, 0, STREAM(stream)>>>(lm, ldv, V, Nl, label_lens, B, U1, part);
    PK_CHECK_LAUNCH(); count_launch();
    smooth_q_finish_kernel<<<col_blocks, 256, 0, STREAM(stream)>>>(part, chunks, ldv, V, label_lens, B, logq);
    PK_CHECK_LAUNCH(); count_launch();
    smooth_lse_kernel<<<B * T, 256, 0, STREAM(stream)>>>(am, ldv, V, am_max, logq, frame_lens, 0, T, Na);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_simple_tables_smooth(const float* am, const float* lm, int ldv, const float* am_max, const float* lm_max,
                                            const float* S, int ld_s, const int* labels, int ld_labels, const int* frame_lens,
                                            const int* label_lens, int B, int T, int U1, const float* Nl, const float* logq, const float* Na,
                                            float lm_only_scale, float am_only_scale, float* lpb_skew, float* lpl_skew, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(Nl && logq && Na, "null pointer");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && ld_s >= U1, "bad dims");
    PK_CHECK_ARG(smooth_scales_ok(lm_only_scale, am_only_scale), "need lm_only_scale >= 0, am_only_scale >= 0, their sum < 1");
    const float mu = 1.f - lm_only_scale - am_only_scale;
    const long long n = (long long)B * T * U1;
    simple_tables_kernel<true><<<grid_of(n), 256, 0, STREAM(stream)>>>(am, lm, ldv, am_max, lm_max, S, ld_s, labels, ld_labels, frame_lens,
                                                                        label_lens, B, T, U1, lpb_skew, lpl_skew, Nl, logq, Na, mu,
                                                                        lm_only_scale, am_only_scale);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_simple_w(const float* gb, const float* gl, const float* S, int ld_s, const int* frame_lens, const int* label_lens,
                                const float* scale, int B, int T, int U1, void* w_hi, void* w_lo, int ld_w, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && ld_s >= U1 && ld_w >= U1 && ld_w % 8 == 0, "bad dims (ld_w >= U1, ld_w % 8 == 0)");
    const long long n = (long long)B * T * ld_w;
    simple_w_kernel<<<grid_of(n), 256, 0, STREAM(stream)>>>(gb, gl, S, ld_s, frame_lens, label_lens, scale, B, T, U1,
                                                             (__nv_bfloat16*)w_hi, (__nv_bfloat16*)w_lo, ld_w);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_simple_grad(const float* src, int ldv, int V, const float* rmax, const float* G, int ld_g, int n_g, int axis,
                                   const float* gb, const float* gl, const int* labels, int ld_labels, const int* frame_lens,
                                   const int* label_lens, const float* scale, int B, int T, int U1, void* out, int out_dtype, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(axis == 0 || axis == 1, "axis must be 0 (rows over t) or 1 (rows over u)");
    PK_CHECK_ARG(out_dtype == PK_F32 || out_dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && V > 0 && ldv >= V && ld_g >= ldv && n_g >= (axis == 0 ? T : U1), "bad dims");
    const size_t smem = (size_t)ldv * 4;
    PK_CHECK_ARG(smem <= 200 * 1024, "ldv too large for the shared-memory row (ldv <= 51200)");
    const int rows = B * (axis == 0 ? T : U1);
    if (out_dtype == PK_BF16) {
        static bool cfg = false;
        if (!cfg) { PK_CHECK_CUDA(cudaFuncSetAttribute(simple_grad_kernel<__nv_bfloat16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); cfg = true; }
        simple_grad_kernel<__nv_bfloat16, false><<<rows, 256, smem, STREAM(stream)>>>(src, ldv, V, rmax, G, ld_g, n_g, axis, gb, gl, labels, ld_labels,
                                                                                      frame_lens, label_lens, scale, T, U1, (__nv_bfloat16*)out);
    } else {
        static bool cfg = false;
        if (!cfg) { PK_CHECK_CUDA(cudaFuncSetAttribute(simple_grad_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); cfg = true; }
        simple_grad_kernel<float, false><<<rows, 256, smem, STREAM(stream)>>>(src, ldv, V, rmax, G, ld_g, n_g, axis, gb, gl, labels, ld_labels,
                                                                              frame_lens, label_lens, scale, T, U1, (float*)out);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_simple_grad_smooth(const float* src, int ldv, int V, const float* rmax, const float* G, int ld_g, int n_g, int axis,
                                          const float* gb, const float* gl, const int* labels, int ld_labels, const int* frame_lens,
                                          const int* label_lens, const float* scale, const float* logq, const float* lse,
                                          float lm_only_scale, float am_only_scale, int B, int T, int U1, void* out, int out_dtype,
                                          void* stream) {
    using namespace pk;
    PK_CHECK_ARG(axis == 0 || axis == 1, "axis must be 0 (rows over t) or 1 (rows over u)");
    PK_CHECK_ARG(out_dtype == PK_F32 || out_dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(lse && (axis == 1 || logq), "null pointer (lse; logq on axis 0)");
    PK_CHECK_ARG(smooth_scales_ok(lm_only_scale, am_only_scale), "need lm_only_scale >= 0, am_only_scale >= 0, their sum < 1");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && V > 0 && ldv >= V && ld_g >= ldv && n_g >= (axis == 0 ? T : U1), "bad dims");
    const size_t smem = (size_t)ldv * 4;
    PK_CHECK_ARG(smem <= 200 * 1024, "ldv too large for the shared-memory row (ldv <= 51200)");
    const int rows = B * (axis == 0 ? T : U1);
    const float mu = 1.f - lm_only_scale - am_only_scale, lam = axis == 0 ? am_only_scale : lm_only_scale;
    const float* lq = axis == 0 ? logq : nullptr;
    if (out_dtype == PK_BF16) {
        static bool cfg = false;
        if (!cfg) { PK_CHECK_CUDA(cudaFuncSetAttribute(simple_grad_kernel<__nv_bfloat16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); cfg = true; }
        simple_grad_kernel<__nv_bfloat16, true><<<rows, 256, smem, STREAM(stream)>>>(src, ldv, V, rmax, G, ld_g, n_g, axis, gb, gl, labels, ld_labels,
                                                                                     frame_lens, label_lens, scale, T, U1, (__nv_bfloat16*)out,
                                                                                     lq, lse, mu, lam);
    } else {
        static bool cfg = false;
        if (!cfg) { PK_CHECK_CUDA(cudaFuncSetAttribute(simple_grad_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); cfg = true; }
        simple_grad_kernel<float, true><<<rows, 256, smem, STREAM(stream)>>>(src, ldv, V, rmax, G, ld_g, n_g, axis, gb, gl, labels, ld_labels,
                                                                             frame_lens, label_lens, scale, T, U1, (float*)out, lq, lse, mu, lam);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_rnnt_prune_bounds(const float* ga, const float* gb, const int* frame_lens, const int* label_lens, int B, int T, int U1,
                                    int R, int* bounds, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(ga && frame_lens && label_lens && bounds, "null pointer");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0, "bad dims");
    PK_CHECK_ARG(R >= 2, "prune range R must be >= 2");
    PK_CHECK_ARG((long long)T * 4 <= 48 * 1024, "T too large for the bounds kernel (T <= 12288)");
    prune_bounds_kernel<<<B, 256, T * 4, STREAM(stream)>>>(ga, gb, frame_lens, label_lens, T, U1, R, bounds);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_joint_gate_pruned_fwd(const void* ex, const void* py, const int* bounds, void* h, int dtype, int B, int T, int U1, int R,
                                        int H, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(dtype == PK_F32 || dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && R >= 1 && H > 0, "bad dims");
    if (dtype == PK_BF16)
        gate_pruned_fwd_kernel<__nv_bfloat16><<<B * T, 128, 0, STREAM(stream)>>>((const __nv_bfloat16*)ex, (const __nv_bfloat16*)py, bounds,
                                                                                (__nv_bfloat16*)h, T, U1, R, H);
    else
        gate_pruned_fwd_kernel<float><<<B * T, 128, 0, STREAM(stream)>>>((const float*)ex, (const float*)py, bounds, (float*)h, T, U1, R, H);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_joint_gate_pruned_bwd(const void* ex, const void* py, const int* bounds, const void* dh, void* dex, void* dpy, int dtype,
                                        int B, int T, int U1, int R, int H, void* stream) {
    using namespace pk;
    PK_CHECK_ARG(dtype == PK_F32 || dtype == PK_BF16, "bad dtype");
    PK_CHECK_ARG(B > 0 && T > 0 && U1 > 0 && R >= 1 && H > 0, "bad dims");
    if (dtype == PK_BF16) {
        using TT = __nv_bfloat16;
        gate_pruned_bwd_ex_kernel<TT><<<B * T, 128, 0, STREAM(stream)>>>((const TT*)ex, (const TT*)py, bounds, (const TT*)dh, (TT*)dex, T, U1, R, H);
        PK_CHECK_LAUNCH(); count_launch();
        gate_pruned_bwd_py_kernel<TT><<<B * U1, 128, 0, STREAM(stream)>>>((const TT*)ex, (const TT*)py, bounds, (const TT*)dh, (TT*)dpy, T, U1, R, H);
    } else {
        using TT = float;
        gate_pruned_bwd_ex_kernel<TT><<<B * T, 128, 0, STREAM(stream)>>>((const TT*)ex, (const TT*)py, bounds, (const TT*)dh, (TT*)dex, T, U1, R, H);
        PK_CHECK_LAUNCH(); count_launch();
        gate_pruned_bwd_py_kernel<TT><<<B * U1, 128, 0, STREAM(stream)>>>((const TT*)ex, (const TT*)py, bounds, (const TT*)dh, (TT*)dpy, T, U1, R, H);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
