// Incremental step of the convolutional-transformer prediction net inside the device beam search (decoder/transducer_decoder.py:
// 117-120,151-171,188-202): instead of re-running the whole partial hypothesis through the network every beam step, each row
// computes only its newest position against a cache of the per-position state that never changes once written.
//
// The prediction net is causal (trainer/model/rnnt_conv_transformer_lm.py:59-80): the output at position p of [blk, y1..yp] reads
//   * per layer l, the causal Conv1d(k=5) taps = the layer's inputs at positions p-4..p (zero before 0), and
//   * per layer l, the attention keys / values of positions 0..p.
// So a pool entry per position holds, for every layer, its K and V rows and (l >= 1) the layer's input; layer 0's input is the
// token's embedding row, gathered from the table.  Entries are written once and never move: entry 0 is the shared SOS position,
// entry 1 + s*rows + row the position computed by `row` at beam step s.  A slot table [2][rows][S1] (ping-pong by step parity, like
// hyp_tok) maps a row's positions to entries; pk_beam_xf_slots reorders it with the back-pointers after each advance, so the rows
// of one utterance share their common prefix's entries.
//
// Every kernel reads the step from step_ctx and the lengths from hyp_len (nothing step-dependent is an argument: the step is
// replayed from a CUDA graph).  All rows are computed; rows whose input token is blank, EOS or done are masked at the writes.
#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

constexpr int XF_TAPS = 5;          // Conv1d kernel size of the reference prediction net
constexpr int XF_DH = 64;           // head size the attention kernel is written for (the reference builds d_model 512 / 8 heads)

struct XfState {
    const int* next_ys;
    const int* step;
    const int* hyp_tok;
    const int* hyp_len;
    int* slot;
    long long n_entries;
    int blk, rows, S1, layers, D, init;
};

struct XfRow {
    bool active;
    int p, par;
    long long entry;
};

// the position a row computes in this launch (see pk_beam_xf_state in include/pika_b200.h)
PK_DEVICE XfRow xf_row(const XfState& c, int row) {
    XfRow r{false, 0, 0, 0};
    if (c.init) { r.active = row == 0; return r; }
    if (c.step[1] == 0) return r;                                                  // the loop has ended: every kernel is a no-op
    const int s = c.step[0];
    r.par = s & 1;
    r.p = c.hyp_len[r.par * c.rows + row];
    r.entry = 1 + (long long)s * c.rows + row;
    r.active = c.next_ys[(long long)s * c.rows + row] > c.blk && r.p < c.S1 && r.entry < c.n_entries;
    return r;
}
PK_DEVICE const int* xf_slots(const XfState& c, const XfRow& r, int row) { return c.slot + ((long long)r.par * c.rows + row) * c.S1; }
// pool entry e, layer l, part w (0 = K, 1 = V, 2 = the layer's input)
template <typename T> PK_DEVICE T* xf_pool(T* pool, const XfState& c, long long e, int l, int w) {
    return pool + ((e * c.layers + l) * 3 + w) * c.D;
}

// ------------------------------------------------------------------------------------ conv taps
// out[row] = [x(p-4) | x(p-3) | ... | x(p)], each tap ldc wide (channels past C zero), x(j) = 0 for j < 0.  Layer 0: x(j) is the
// embedding row of the token at position j (blk at 0, hyp_tok[j-1] after); layer l >= 1: x(p) is x_cur[row] (the previous
// layer's output just computed, which this kernel also stores into the row's pool entry) and x(j < p) comes from the pool.
template <typename T>
__global__ void xf_taps_kernel(XfState c, T* pool, int l, const float* __restrict__ embed, int E, const T* __restrict__ x_cur, int ldc,
                               T* __restrict__ out) {
    const int row = blockIdx.x;
    const XfRow r = xf_row(c, row);
    T* o = out + (long long)row * XF_TAPS * ldc;
    if (!r.active) {
        for (int i = threadIdx.x; i < XF_TAPS * ldc; i += blockDim.x) o[i] = from_f32<T>(0.f);
        return;
    }
    const int C = (l == 0) ? E : c.D;
    const int* tok = c.hyp_tok + ((long long)r.par * c.rows + row) * c.S1;
    const int* slots = xf_slots(c, r, row);
    const T* xc = x_cur + (long long)row * c.D;
    if (l > 0) {
        T* dst = xf_pool(pool, c, r.entry, l, 2);
        for (int ch = threadIdx.x; ch < c.D; ch += blockDim.x) dst[ch] = xc[ch];
    } else if (!c.init && threadIdx.x == 0) {
        c.slot[((long long)r.par * c.rows + row) * c.S1 + r.p] = (int)r.entry;
    }
    for (int i = threadIdx.x; i < XF_TAPS * ldc; i += blockDim.x) {
        const int k = i / ldc, ch = i - k * ldc;
        const int j = r.p - (XF_TAPS - 1) + k;
        T v = from_f32<T>(0.f);
        if (j >= 0 && ch < C) {
            if (l == 0) v = from_f32<T>(embed[(long long)(j == 0 ? c.blk : tok[j - 1]) * E + ch]);
            else if (j == r.p) v = xc[ch];
            else v = xf_pool(pool, c, slots[j], l, 2)[ch];
        }
        o[i] = v;
    }
}

// ------------------------------------------------------------------------------------ single-query attention
template <typename T> PK_DEVICE void load8(const T* p, float (&v)[8]);
template <> PK_DEVICE void load8<float>(const float* p, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> PK_DEVICE void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    v[0] = bf16lo(u.x); v[1] = bf16hi(u.x); v[2] = bf16lo(u.y); v[3] = bf16hi(u.y);
    v[4] = bf16lo(u.z); v[5] = bf16hi(u.z); v[6] = bf16lo(u.w); v[7] = bf16hi(u.w);
}

// One CTA per row, one warp per head.  The new position's K / V (columns D.. and 2D.. of the row's fused QKV) are stored into the
// row's pool entry; the query attends over positions 0..p through the slot table, 32 keys per round (lane i scores key j0 + i with a
// full 64-wide dot product), with an fp32 online softmax; then every lane accumulates its two output columns over the round's keys.
// Relative positions (max_rel = m > 0, trainer/model/modules/multi_headed_attn.py:186-229): key j has bucket clip(j - p, -m, m) + m of
// the table R shared by keys and values, so the score adds (alpha q) . R[bucket] and the output adds p_j R[bucket].
template <typename T>
__global__ void xf_attn_kernel(XfState c, T* pool, int l, const T* __restrict__ qkv, const float* __restrict__ rel, int max_rel, float alpha,
                               T* __restrict__ out) {
    const int row = blockIdx.x, h = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ __align__(16) float s_q[32][XF_DH];
    const XfRow r = xf_row(c, row);
    T* o = out + (long long)row * c.D + h * XF_DH + 2 * lane;
    if (!r.active) {
        o[0] = o[1] = from_f32<T>(0.f);
        return;
    }
    const T* q = qkv + (long long)row * 3 * c.D + h * XF_DH;
    const T* k_new = q + c.D;                          // V follows K at +D in both the QKV row and a pool entry
    s_q[h][2 * lane] = alpha * to_f32(q[2 * lane]);
    s_q[h][2 * lane + 1] = alpha * to_f32(q[2 * lane + 1]);
    T* ent = xf_pool(pool, c, r.entry, l, 0) + h * XF_DH;
    ent[2 * lane] = k_new[2 * lane];
    ent[2 * lane + 1] = k_new[2 * lane + 1];
    ent[c.D + 2 * lane] = k_new[c.D + 2 * lane];
    ent[c.D + 2 * lane + 1] = k_new[c.D + 2 * lane + 1];
    __syncwarp();
    const int* slots = xf_slots(c, r, row);
    const int p = r.p;
    auto bucket = [&](int j) { return max(j - p, -max_rel) + max_rel; };
    auto k_row = [&](int j, int e) -> const T* { return j == p ? k_new : xf_pool(pool, c, e, l, 0) + h * XF_DH; };
    float m_run = -INFINITY, l_run = 0.f, a0 = 0.f, a1 = 0.f;
    for (int j0 = 0; j0 <= p; j0 += 32) {
        const int j = j0 + lane;
        const bool valid = j <= p;
        const int e = (valid && j < p) ? slots[j] : 0;
        float s = -INFINITY;
        if (valid) {
            const T* kr = k_row(j, e);
            float dot = 0.f;
#pragma unroll
            for (int d0 = 0; d0 < XF_DH; d0 += 8) {
                float kv[8];
                load8<T>(kr + d0, kv);
#pragma unroll
                for (int i = 0; i < 8; ++i) dot = fmaf(s_q[h][d0 + i], kv[i], dot);
            }
            if (max_rel > 0) {
                const float* rr = rel + (long long)bucket(j) * XF_DH;
                float dr = 0.f;
#pragma unroll 8
                for (int d = 0; d < XF_DH; ++d) dr = fmaf(s_q[h][d], rr[d], dr);
                dot += dr;
            }
            s = dot;
        }
        float mx = s;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float m_new = fmaxf(m_run, mx);
        const float corr = expf(m_run - m_new);                                   // 0 in the first round (m_run = -inf)
        const float pj = valid ? expf(s - m_new) : 0.f;
        float ps = pj;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
        l_run = l_run * corr + ps;
        a0 *= corr;
        a1 *= corr;
        m_run = m_new;
        const int n = min(32, p + 1 - j0);
        for (int i = 0; i < n; ++i) {
            const float pi = __shfl_sync(0xffffffffu, pj, i);
            const int ei = __shfl_sync(0xffffffffu, e, i);
            const T* vr = k_row(j0 + i, ei) + c.D;
            a0 = fmaf(pi, to_f32(vr[2 * lane]), a0);
            a1 = fmaf(pi, to_f32(vr[2 * lane + 1]), a1);
            if (max_rel > 0) {
                const float* rr = rel + (long long)bucket(j0 + i) * XF_DH;
                a0 = fmaf(pi, rr[2 * lane], a0);
                a1 = fmaf(pi, rr[2 * lane + 1], a1);
            }
        }
    }
    const float inv = 1.f / l_run;
    o[0] = from_f32<T>(a0 * inv);
    o[1] = from_f32<T>(a1 * inv);
}

// ------------------------------------------------------------------------------------ state update
// h[row] = x[row] on the rows that computed a position (init: every row takes row 0's output, the SOS state)
template <typename T>
__global__ void xf_select_kernel(XfState c, const T* __restrict__ x, T* __restrict__ h, int H) {
    const int row = blockIdx.x;
    const XfRow r = xf_row(c, row);
    if (!c.init && !r.active) return;
    const T* src = x + (long long)(c.init ? 0 : row) * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) h[(long long)row * H + i] = src[i];
}

// after the advance of step s: new beam k continues row src = prev_ks[s][k] (or itself when it finished, as the hypothesis update
// does), so its positions 0..hyp_len[s&1][src] are src's
__global__ void xf_slots_kernel(XfState c, const int* __restrict__ prev_ks, int K) {
    const int row = blockIdx.x;
    if (c.step[1] == 0) return;
    const int s = c.step[0], po = s & 1, pn = po ^ 1;
    const int src = c.next_ys[(long long)(s + 1) * c.rows + row] == -1 ? row : (row / K) * K + prev_ks[(long long)s * c.rows + row];
    const int n = min(c.hyp_len[po * c.rows + src], c.S1 - 1);
    const int* from = c.slot + ((long long)po * c.rows + src) * c.S1;
    int* to = c.slot + ((long long)pn * c.rows + row) * c.S1;
    for (int q = threadIdx.x; q <= n; q += blockDim.x) to[q] = from[q];
}
}  // namespace pk

using namespace pk;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

static int xf_state(const pk_beam_xf_state* st, XfState& c) {
    PK_CHECK_ARG(st != nullptr && st->next_ys && st->step_ctx && st->hyp_tok && st->hyp_len && st->slot && st->pool, "null beam_xf state");
    PK_CHECK_ARG(st->rows > 0 && st->S1 > 0 && st->layers > 0 && st->n_entries > 0, "empty beam_xf state");
    PK_CHECK_ARG(st->D > 0 && st->D % 8 == 0, "d_model must be a positive multiple of 8");
    PK_CHECK_ARG(st->dtype == PK_BF16 || st->dtype == PK_F32, "dtype must be PK_BF16 or PK_F32");
    c = XfState{st->next_ys, st->step_ctx, st->hyp_tok, st->hyp_len, st->slot, st->n_entries, st->blk, st->rows, st->S1, st->layers, st->D,
                st->init};
    return 0;
}
#define XF_STATE(st, c)                          \
    XfState c;                                   \
    if (xf_state(st, c) != 0) return -1

extern "C" int pk_beam_xf_taps(const pk_beam_xf_state* st, int layer, const float* embed, int E, const void* x_cur, void* taps, int ldc,
                               void* stream) {
    XF_STATE(st, c);
    PK_CHECK_ARG(layer >= 0 && layer < st->layers, "layer out of range");
    PK_CHECK_ARG(layer > 0 || (embed != nullptr && E > 0 && ldc >= E), "layer 0 needs the embedding table and ldc >= E");
    PK_CHECK_ARG(layer == 0 || (x_cur != nullptr && ldc >= st->D), "layers >= 1 need x_cur and ldc >= d_model");
    PK_CHECK_ARG(ldc % 8 == 0 && taps != nullptr, "ldc must be a multiple of 8");
    if (st->dtype == PK_BF16)
        xf_taps_kernel<__nv_bfloat16><<<st->rows, 128, 0, ST(stream)>>>(c, (__nv_bfloat16*)st->pool, layer, embed, E,
                                                                       (const __nv_bfloat16*)x_cur, ldc, (__nv_bfloat16*)taps);
    else
        xf_taps_kernel<float><<<st->rows, 128, 0, ST(stream)>>>(c, (float*)st->pool, layer, embed, E, (const float*)x_cur, ldc, (float*)taps);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_beam_xf_attn(const pk_beam_xf_state* st, int layer, const void* qkv, int heads, const float* rel, int max_rel, void* out,
                               void* stream) {
    XF_STATE(st, c);
    PK_CHECK_ARG(layer >= 0 && layer < st->layers, "layer out of range");
    PK_CHECK_ARG(heads > 0 && heads * XF_DH == st->D, "the decode attention needs a head size of 64 (d_model == 64 * heads)");
    PK_CHECK_ARG(heads <= 32, "at most 32 heads");
    PK_CHECK_ARG(max_rel >= 0 && (max_rel == 0 || rel != nullptr), "max_rel > 0 needs the relative-position table");
    PK_CHECK_ARG(qkv != nullptr && out != nullptr, "null qkv / out");
    const float alpha = 1.f / sqrtf((float)XF_DH);
    if (st->dtype == PK_BF16)
        xf_attn_kernel<__nv_bfloat16><<<st->rows, heads * 32, 0, ST(stream)>>>(c, (__nv_bfloat16*)st->pool, layer, (const __nv_bfloat16*)qkv, rel,
                                                                              max_rel, alpha, (__nv_bfloat16*)out);
    else
        xf_attn_kernel<float><<<st->rows, heads * 32, 0, ST(stream)>>>(c, (float*)st->pool, layer, (const float*)qkv, rel, max_rel, alpha,
                                                                      (float*)out);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_beam_xf_select(const pk_beam_xf_state* st, const void* x, void* h, int H, void* stream) {
    XF_STATE(st, c);
    PK_CHECK_ARG(x != nullptr && h != nullptr && H > 0, "null x / h or H <= 0");
    if (st->dtype == PK_BF16)
        xf_select_kernel<__nv_bfloat16><<<st->rows, 128, 0, ST(stream)>>>(c, (const __nv_bfloat16*)x, (__nv_bfloat16*)h, H);
    else
        xf_select_kernel<float><<<st->rows, 128, 0, ST(stream)>>>(c, (const float*)x, (float*)h, H);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_beam_xf_slots(const pk_beam_xf_state* st, const int* prev_ks, int K, void* stream) {
    XF_STATE(st, c);
    PK_CHECK_ARG(prev_ks != nullptr && K > 0 && st->rows % K == 0, "prev_ks / beam size");
    xf_slots_kernel<<<st->rows, 128, 0, ST(stream)>>>(c, prev_ks, K);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
