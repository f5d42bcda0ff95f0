// Memory-bound kernels around the GEMMs: casts/splits, BatchNorm, LayerNorm, attention softmax,
// dropout, column sums, gated joint, LSTM cell, embedding.  All are HBM-bound: 16-byte accesses,
// threads along the contiguous channel axis, grids sized in multiples of the SM count.
// Activations are templated on T = bf16 (production) | f32 (fp32-class parity mode).
#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

template <typename T> struct V8 {};   // 8 consecutive elements
template <> struct V8<__nv_bfloat16> {
    struct Raw { uint4 q; };                                    // the 16 bytes as loaded (kept packed while a prefetch is in flight)
    PK_DEVICE static Raw load_raw(const __nv_bfloat16* p) { return Raw{*reinterpret_cast<const uint4*>(p)}; }
    PK_DEVICE static void unpack(const Raw& r, float (&f)[8]) {
        f[0] = bf16lo(r.q.x); f[1] = bf16hi(r.q.x); f[2] = bf16lo(r.q.y); f[3] = bf16hi(r.q.y);
        f[4] = bf16lo(r.q.z); f[5] = bf16hi(r.q.z); f[6] = bf16lo(r.q.w); f[7] = bf16hi(r.q.w);
    }
    PK_DEVICE static void load(const __nv_bfloat16* p, float (&f)[8]) {
        const uint4 q = *reinterpret_cast<const uint4*>(p);
        f[0] = bf16lo(q.x); f[1] = bf16hi(q.x); f[2] = bf16lo(q.y); f[3] = bf16hi(q.y);
        f[4] = bf16lo(q.z); f[5] = bf16hi(q.z); f[6] = bf16lo(q.w); f[7] = bf16hi(q.w);
    }
    PK_DEVICE static void store(__nv_bfloat16* p, const float (&f)[8]) {
        *reinterpret_cast<uint4*>(p) =
            make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
    }
};
template <> struct V8<float> {
    struct Raw { float4 a, b; };
    PK_DEVICE static Raw load_raw(const float* p) { return Raw{*reinterpret_cast<const float4*>(p), *reinterpret_cast<const float4*>(p + 4)}; }
    PK_DEVICE static void unpack(const Raw& r, float (&f)[8]) {
        f[0] = r.a.x; f[1] = r.a.y; f[2] = r.a.z; f[3] = r.a.w; f[4] = r.b.x; f[5] = r.b.y; f[6] = r.b.z; f[7] = r.b.w;
    }
    PK_DEVICE static void load(const float* p, float (&f)[8]) {
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
        f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    }
    PK_DEVICE static void store(float* p, const float (&f)[8]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
};

static inline int grid_for(long long work_items, int per_cta, int waves = 8) {
    long long g = (work_items + per_cta - 1) / per_cta;
    long long cap = (long long)num_sms() * waves;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

#define PK_DISPATCH_T(dtype, ...)                                         \
    if ((dtype) == PK_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }     \
    else { using T = float; __VA_ARGS__; }

// =============================================================================== cast / split
// dst_hi[r, c] = bf16(scale * src[r, c]); dst_lo = bf16(scale*src - hi) (optional); columns
// [cols, cols_pad) of dst are zero-filled.  src is f32 or bf16 (strided rows).
template <typename S>
__global__ void cast_split_kernel(const S* __restrict__ src, long long ld_src, __nv_bfloat16* __restrict__ hi,
                                  __nv_bfloat16* __restrict__ lo, long long ld_dst, long long rows, int cols, int cols_pad,
                                  float scale) {
    const long long total = rows * cols_pad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cols_pad;
        const int c = (int)(i - r * cols_pad);
        float v = 0.f;
        if (c < cols) v = to_f32<S>(src[r * ld_src + c]) * scale;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi[r * ld_dst + c] = h;
        if (lo) lo[r * ld_dst + c] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// =============================================================================== column statistics
// sums[c] += sum_r f(x[r,c]); sums2[c] += sum_r x[r,c]*g[r,c]  (g = x for BN stats, x_hat for BN/LN bwd)
// Block: 128 threads x 8 channels = 1024 channels per pass; rows split across blockIdx.y.
// MODE 0: (sum x, sum x^2); 1: (sum dy, sum dy*xhat) with xhat=(x-mean)*rstd;
// 2: (sum d, sum d^2) with d = x - x[0,c]: the BN statistics.  Shifting by a value of the channel keeps s2/n - (s1/n)^2 accurate when
//    the channel's mean is large against its spread (an almost-always-on ReLU channel): unshifted f32 sums lose that variance to
//    cancellation.  Every row slice shifts by the same row 0, so the partials still add.
template <typename T, int MODE>
__global__ void __launch_bounds__(128, 4) colstats_kernel(const T* __restrict__ x, const T* __restrict__ aux, long long rows, int C,
                                                       const float* __restrict__ mean, const float* __restrict__ rstd,
                                                       float* __restrict__ s1) {
    const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
    if (c0 >= C) return;
    const long long rows_per = (rows + gridDim.y - 1) / gridDim.y;
    const long long r0 = (long long)blockIdx.y * rows_per;
    const long long r1 = min(rows, r0 + rows_per);
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    float mu[8], rs[8], piv[8];
    if (MODE == 1) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { mu[e] = mean[c0 + e]; rs[e] = rstd[c0 + e]; }
    }
    if (MODE == 2) V8<T>::load(x + c0, piv);
    constexpr int UR = 8;                       // independent 16-byte loads in flight per thread
    long long r = r0;
    for (; r + UR <= r1; r += UR) {
        float f[UR][8], g[UR][8];
#pragma unroll
        for (int k = 0; k < UR; ++k) {
            V8<T>::load(x + (r + k) * C + c0, f[k]);
            if (MODE == 1) V8<T>::load(aux + (r + k) * C + c0, g[k]);        // aux = BN input x; f = dy
        }
#pragma unroll
        for (int k = 0; k < UR; ++k) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if (MODE == 2) f[k][e] -= piv[e];
                a[e] += f[k][e];
                b[e] += (MODE == 1) ? f[k][e] * (g[k][e] - mu[e]) * rs[e] : f[k][e] * f[k][e];
            }
        }
    }
    for (; r < r1; ++r) {
        float f[8], g[8];
        V8<T>::load(x + r * C + c0, f);
        if (MODE == 1) V8<T>::load(aux + r * C + c0, g);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            if (MODE == 2) f[e] -= piv[e];
            a[e] += f[e];
            b[e] += (MODE == 1) ? f[e] * (g[e] - mu[e]) * rs[e] : f[e] * f[e];
        }
    }
    // partial sums of this row-slice: part[(blockIdx.y * 2 + {0,1}) * C + c]
    float* p1 = s1 + (long long)(blockIdx.y * 2) * C + c0;
    float* p2 = p1 + C;
    *reinterpret_cast<float4*>(p1) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(p1 + 4) = make_float4(a[4], a[5], a[6], a[7]);
    *reinterpret_cast<float4*>(p2) = make_float4(b[0], b[1], b[2], b[3]);
    *reinterpret_cast<float4*>(p2 + 4) = make_float4(b[4], b[5], b[6], b[7]);
}
// out1[c] = sum_y part[y][0][c], out2[c] = sum_y part[y][1][c]   (fixed order: deterministic)
// block = 32 columns x 8 y-groups
__global__ void __launch_bounds__(256) colstats_reduce_kernel(const float* __restrict__ part, int gy, int C, float* __restrict__ out1,
                                                              float* __restrict__ out2) {
    __shared__ float sa[8][33], sb[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx;
    float a = 0.f, b = 0.f;
    if (c < C) {
        for (int y = ty; y < gy; y += 8) { a += part[(long long)(y * 2) * C + c]; b += part[(long long)(y * 2 + 1) * C + c]; }
    }
    sa[ty][tx] = a; sb[ty][tx] = b;
    __syncthreads();
    if (ty == 0 && c < C) {
#pragma unroll
        for (int k = 1; k < 8; ++k) { a += sa[k][tx]; b += sb[k][tx]; }
        out1[c] = a;
        if (out2) out2[c] = b;
    }
}

// mean/rstd from the shifted sums of colstats MODE 2 (s1 = sum d, s2 = sum d^2, d = x - x[0,c]); optional running-stat update
// (nn.BatchNorm1d: unbiased var, the caller's momentum)
template <typename T>
__global__ void bn_finalize_kernel(const T* __restrict__ x, const float* __restrict__ s1, const float* __restrict__ s2, long long rows,
                                   int C, float eps, float momentum, float* __restrict__ mean, float* __restrict__ rstd,
                                   float* __restrict__ run_mean, float* __restrict__ run_var) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float n = (float)rows;
    const float d = s1[c] / n;                                  // mean - x[0,c]
    float var = s2[c] / n - d * d;
    var = fmaxf(var, 0.f);
    const float m = to_f32<T>(x[c]) + d;
    mean[c] = m;
    rstd[c] = rsqrtf(var + eps);
    if (run_mean) {
        run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * m;
        const float unb = rows > 1 ? var * n / (n - 1.f) : var;
        run_var[c] = (1.f - momentum) * run_var[c] + momentum * unb;
    }
}
__global__ void bn_eval_stats_kernel(const float* __restrict__ run_mean, const float* __restrict__ run_var, int C, float eps,
                                     float* __restrict__ mean, float* __restrict__ rstd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mean[c] = run_mean[c];
    rstd[c] = rsqrtf(run_var[c] + eps);
}

// Column-resident streaming kernels: a thread owns 8 consecutive channels (its per-channel coefficients live in registers) and
// walks a slice of the rows with UR 16-byte loads in flight -- no per-element coefficient loads, no index arithmetic in the loop.
// Block = 128 threads = 1024 channels (gridDim.x covers C), gridDim.y slices the rows.
//
// y = (x - mean) * rstd * w + b  ==  x * sc + sh
template <typename T>
__global__ void __launch_bounds__(128) bn_apply_kernel(const T* __restrict__ x, T* __restrict__ y, long long rows, int C,
                                                       const float* __restrict__ mean, const float* __restrict__ rstd,
                                                       const float* __restrict__ w, const float* __restrict__ b) {
    const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
    if (c0 >= C) return;
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        sc[e] = rstd[c0 + e] * w[c0 + e];
        sh[e] = b[c0 + e] - mean[c0 + e] * sc[e];
    }
    const long long rows_per = (rows + gridDim.y - 1) / gridDim.y;
    const long long r0 = (long long)blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
    constexpr int UR = 8;
    long long r = r0;
    for (; r + UR <= r1; r += UR) {
        float f[UR][8];
#pragma unroll
        for (int k = 0; k < UR; ++k) V8<T>::load(x + (r + k) * C + c0, f[k]);
#pragma unroll
        for (int k = 0; k < UR; ++k) {
#pragma unroll
            for (int e = 0; e < 8; ++e) f[k][e] = fmaf(f[k][e], sc[e], sh[e]);
            V8<T>::store(y + (r + k) * C + c0, f[k]);
        }
    }
    for (; r < r1; ++r) {
        float f[8];
        V8<T>::load(x + r * C + c0, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf(f[e], sc[e], sh[e]);
        V8<T>::store(y + r * C + c0, f);
    }
}

// BN backward (train): dx = w*rstd*(dy - sdy/n - xhat*sdyx/n) == A*dy + Bx*x + C0 per channel; optionally masked by
// relu_mask (x > 0, x being the BN input = ReLU output, so this also back-propagates through the ReLU).
// eval mode (sdy == nullptr): dx = w*rstd*dy.
template <typename T>
__global__ void __launch_bounds__(128) bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dx,
                                                           long long rows, int C, const float* __restrict__ mean,
                                                           const float* __restrict__ rstd, const float* __restrict__ w,
                                                           const float* __restrict__ sdy, const float* __restrict__ sdyx,
                                                           int relu_mask) {
    const int c0 = (blockIdx.x * 128 + threadIdx.x) * 8;
    if (c0 >= C) return;
    const float inv_n = 1.f / (float)rows;
    float ca[8], cb[8], cc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int c = c0 + e;
        const float a = w[c] * rstd[c];
        ca[e] = a;
        if (sdy) {
            const float k = rstd[c] * sdyx[c] * inv_n;         // coefficient of xhat's (x - mean)
            cb[e] = -a * k;
            cc[e] = a * (mean[c] * k - sdy[c] * inv_n);
        } else {
            cb[e] = 0.f; cc[e] = 0.f;
        }
    }
    const long long rows_per = (rows + gridDim.y - 1) / gridDim.y;
    const long long r0 = (long long)blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
    constexpr int UR = 4;
    long long r = r0;
    for (; r + UR <= r1; r += UR) {
        float g[UR][8], f[UR][8];
#pragma unroll
        for (int k = 0; k < UR; ++k) { V8<T>::load(dy + (r + k) * C + c0, g[k]); V8<T>::load(x + (r + k) * C + c0, f[k]); }
#pragma unroll
        for (int k = 0; k < UR; ++k) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float d = fmaf(g[k][e], ca[e], fmaf(f[k][e], cb[e], cc[e]));
                g[k][e] = (relu_mask && !(f[k][e] > 0.f)) ? 0.f : d;
            }
            V8<T>::store(dx + (r + k) * C + c0, g[k]);
        }
    }
    for (; r < r1; ++r) {
        float g[8], f[8];
        V8<T>::load(dy + r * C + c0, g);
        V8<T>::load(x + r * C + c0, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float d = fmaf(g[e], ca[e], fmaf(f[e], cb[e], cc[e]));
            g[e] = (relu_mask && !(f[e] > 0.f)) ? 0.f : d;
        }
        V8<T>::store(dx + r * C + c0, g);
    }
}
// (column blocks, row slices) for the two kernels above: enough CTAs for ~8 per SM
static inline dim3 col_grid(long long rows, int C) {
    const int gx = (C + 1023) / 1024;
    long long gy = ((long long)num_sms() * 8 + gx - 1) / gx;
    const long long max_gy = (rows + 15) / 16;                 // at least 16 rows per slice
    if (gy > max_gy) gy = max_gy;
    if (gy < 1) gy = 1;
    return dim3(gx, (unsigned)gy);
}

// =============================================================================== LayerNorm (C <= 1024, C % 8 == 0)
// one warp per row
template <typename T>
__global__ void __launch_bounds__(256) ln_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, long long rows, int C,
                                                     const float* __restrict__ w, const float* __restrict__ b, float eps,
                                                     float* __restrict__ mean_out, float* __restrict__ rstd_out) {
    // one warp per row; C <= 1024: the row lives in registers (lane l owns columns [l*8 + k*256, +8)), x is read exactly once and the
    // next row of the warp is already in flight (packed) while this one is reduced and written
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    typename V8<T>::Raw nx[4];
    if (warp < rows) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { const int c = lane * 8 + k * 256; if (c < C) nx[k] = V8<T>::load_raw(x + warp * C + c); }
    }
    const float invC = 1.f / C;
    for (long long r = warp; r < rows; r += nw) {
        float f[4][8];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) {
                V8<T>::unpack(nx[k], f[k]);
#pragma unroll
                for (int e = 0; e < 8; ++e) s += f[k][e];
            }
        }
        if (r + nw < rows) {
#pragma unroll
            for (int k = 0; k < 4; ++k) { const int c = lane * 8 + k * 256; if (c < C) nx[k] = V8<T>::load_raw(x + (r + nw) * C + c); }
        }
        const float mu = warp_sum(s) * invC;
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) {
#pragma unroll
                for (int e = 0; e < 8; ++e) v += (f[k][e] - mu) * (f[k][e] - mu);
            }
        }
        const float rs = rsqrtf(warp_sum(v) * invC + eps);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) {
#pragma unroll
                for (int e = 0; e < 8; ++e) f[k][e] = (f[k][e] - mu) * rs * __ldg(w + c + e) + __ldg(b + c + e);   // L1-resident
                V8<T>::store(y + r * C + c, f[k]);
            }
        }
        if (lane == 0 && mean_out) { mean_out[r] = mu; rstd_out[r] = rs; }
    }
}

// dx = rstd * (g - mean(g) - xhat * mean(g*xhat)), g = dy*w;  dw[c] += sum dy*xhat, db[c] += sum dy
// Column sums: each lane keeps its own columns in registers across all rows of its warp (C <= 1024),
// warps combine through shared memory, one global atomicAdd per column per CTA.
template <typename T>
__global__ void __launch_bounds__(256) ln_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dx,
                                                     long long rows, int C, const float* __restrict__ w,
                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                     float* __restrict__ dw, float* __restrict__ db) {
    extern __shared__ float sh[];       // dw_part[C], db_part[C]
    float* dwp = sh;
    float* dbp = sh + C;
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sh[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    float aw[4][8], ab[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) { aw[k][e] = 0.f; ab[k][e] = 0.f; }
    float wr[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = lane * 8 + k * 256;
#pragma unroll
        for (int e = 0; e < 8; ++e) wr[k][e] = c < C ? w[c + e] : 0.f;
    }
    typename V8<T>::Raw ng[4], nf[4];                           // the warp's next row, in flight (packed) while this one is processed
    if (warp < rows) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) { ng[k] = V8<T>::load_raw(dy + warp * C + c); nf[k] = V8<T>::load_raw(x + warp * C + c); }
        }
    }
    for (long long r = warp; r < rows; r += nw) {
        const float mu = mean[r], rs = rstd[r];
        float s1 = 0.f, s2 = 0.f;
        float g[4][8], f[4][8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) { V8<T>::unpack(ng[k], g[k]); V8<T>::unpack(nf[k], f[k]); }
        }
        if (r + nw < rows) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int c = lane * 8 + k * 256;
                if (c < C) { ng[k] = V8<T>::load_raw(dy + (r + nw) * C + c); nf[k] = V8<T>::load_raw(x + (r + nw) * C + c); }
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    f[k][e] = (f[k][e] - mu) * rs;              // xhat
                    const float gw = g[k][e] * wr[k][e];
                    s1 += gw; s2 += gw * f[k][e];
                }
            }
        }
        s1 = warp_sum(s1) / C; s2 = warp_sum(s2) / C;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = lane * 8 + k * 256;
            if (c < C) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    o[e] = rs * (g[k][e] * wr[k][e] - s1 - f[k][e] * s2);
                    aw[k][e] += g[k][e] * f[k][e];
                    ab[k][e] += g[k][e];
                }
                V8<T>::store(dx + r * C + c, o);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = lane * 8 + k * 256;
        if (c < C) {
#pragma unroll
            for (int e = 0; e < 8; ++e) { atomicAdd(&dwp[c + e], aw[k][e]); atomicAdd(&dbp[c + e], ab[k][e]); }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
        atomicAdd(&dw[i], dwp[i]);
        atomicAdd(&db[i], dbp[i]);
    }
}

// =============================================================================== attention softmax
// S f32 [rows, ld_s] (first n valid) -> P (T) [rows, ld_p] and Pd = dropout(P); pad columns [n, ld_p) zeroed.
// One warp per row; the row lives in registers (lane l owns columns [l*8 + k*256, +8), k < 4, n <= 1024) and every
// access is a 16/32-byte vector, so S is read exactly once.  ld_s, ld_p multiples of 8.
PK_DEVICE void ld8f(const float* p, float (&f)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T, int SM_CH, bool CHUNK = false>
__global__ void __launch_bounds__(256) softmax_fwd_kernel(const float* __restrict__ S, long long ld_s, T* __restrict__ P,
                                                          T* __restrict__ Pd, long long ld_p, long long rows, int n,
                                                          uint32_t drop_thresh, float drop_scale, uint32_t seed, int q_len = 0,
                                                          int heads = 1, int causal = 0, const uint8_t* __restrict__ key_pad = nullptr,
                                                          int chunk_len = 1, int chunk_off = 0, int left_chunks = -1) {
    // masked form (q_len > 0; the transformer prediction net, trainer/model/rnnt_conv_transformer_lm.py:66-70): row r is query
    // i = r % q_len of sequence r / (heads * q_len); key c is dropped when c > i (causal) or key_pad[seq, c] != 0.  A dropped score
    // becomes -inf where the reference fills -1e18 (multi_headed_attn.py:214-216): both give probability exactly 0 as long as one key
    // survives, which the causal diagonal guarantees.
    // CHUNK (pk_softmax_chunk_fwd; q_len = n, self-attention): query i keeps the keys [chunk_key_lo, chunk_key_hi) of the chunk mask
    // (common.cuh), which always hold i itself.
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        const float* sr = S + r * ld_s;
        float v[SM_CH][8];
        float m = -INFINITY;
        int lim = n, lo = 0;
        const uint8_t* kp = nullptr;
        if (CHUNK) {
            const int i = (int)(r % q_len);
            lo = chunk_key_lo(i, n, chunk_len, chunk_off, left_chunks);
            lim = chunk_key_hi(i, n, chunk_len, chunk_off);
        } else if (q_len > 0) {
            if (causal) lim = min(n, (int)(r % q_len) + 1);
            if (key_pad) kp = key_pad + (r / ((long long)heads * q_len)) * n;
        }
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) ld8f(sr + c0, v[k]);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if (c0 + e >= lim || (CHUNK && c0 + e < lo) || (kp && kp[c0 + e])) v[k][e] = -INFINITY;
                m = fmaxf(m, v[k][e]);
            }
        }
        m = warp_max(m);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < SM_CH; ++k)
#pragma unroll
            for (int e = 0; e < 8; ++e) { v[k][e] = __expf(v[k][e] - m); s += v[k][e]; }
        const float inv = 1.f / warp_sum(s);
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
                float o[8], od[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    o[e] = to_f32<T>(from_f32<T>(v[k][e] * inv));        // dropout acts on the rounded probability
                    od[e] = o[e];
                }
                if (drop_thresh) {                                       // pair mask shared with the fused attention kernels (common.cuh)
                    const uint32_t salt = drop_row_salt((uint64_t)r, seed);
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const uint32_t km = drop_pair(salt, (uint32_t)((c0 >> 1) + e2), drop_thresh);
                        od[2 * e2] = (km & 1u) ? o[2 * e2] * drop_scale : 0.f;
                        od[2 * e2 + 1] = (km & 2u) ? o[2 * e2 + 1] * drop_scale : 0.f;
                    }
                }
                V8<T>::store(P + r * ld_p + c0, o);
                if (Pd != P) V8<T>::store(Pd + r * ld_p + c0, od);
            }
        }
    }
}
// dS[r,c] = P * (dP' - sum_c dP'*P), dP' = dPd * mask * scale; written as T with pad zeroed.
template <typename T, int SM_CH>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(const float* __restrict__ dPd, long long ld_d, const T* __restrict__ P,
                                                          long long ld_p, T* __restrict__ dS, long long rows, int n,
                                                          uint32_t drop_thresh, float drop_scale, uint32_t seed) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        float d[SM_CH][8], pv[SM_CH][8];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
                ld8f(dPd + r * ld_d + c0, d[k]);
                V8<T>::load(P + r * ld_p + c0, pv[k]);
#pragma unroll
                if (drop_thresh) {
                    const uint32_t salt = drop_row_salt((uint64_t)r, seed);
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const uint32_t km = drop_pair(salt, (uint32_t)((c0 >> 1) + e2), drop_thresh);
                        d[k][2 * e2] = (km & 1u) ? d[k][2 * e2] * drop_scale : 0.f;
                        d[k][2 * e2 + 1] = (km & 2u) ? d[k][2 * e2 + 1] * drop_scale : 0.f;
                    }
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    if (c0 + e >= n) { d[k][e] = 0.f; pv[k][e] = 0.f; }
                    dot += d[k][e] * pv[k][e];
                }
            }
        }
        dot = warp_sum(dot);
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = pv[k][e] * (d[k][e] - dot);
                V8<T>::store(dS + r * ld_p + c0, o);
            }
        }
    }
}

// ------------------------------------------------------------------------------- relative positions (Shaw et al.)
// Query i and key j of one sequence share the table row bucket(i, j) = clamp(j - i, -mr, mr) + mr
// (trainer/model/modules/multi_headed_attn.py:9-24).  Along a row the buckets form a band: bucket r in (0, 2mr) is the single key
// j = i - mr + r, bucket 0 collects every j <= i - mr and bucket 2mr every j >= i + mr.  So the gather of the table terms is one
// scalar load per key, and the per-bucket reduction is a shifted copy of the row plus two warp sums -- no atomics, no [T, T, d]
// tensor.  The bucket rows (QR, Pb, G, dSb) are token-major: row (sequence, query, head), the layout of the [B, T, heads*dh]
// activations, so the GEMMs that produce and consume them see plain 2-D matrices.
PK_DEVICE int relpos_bucket(int dist, int mr) { return min(max(dist, -mr), mr) + mr; }

// out[r] = sum of v over keys j < n with bucket(i, j) = r, for r < ld_r (0 for buckets no key reaches and for the padding r > 2mr).
// v holds the row in the softmax kernels' register layout.  Every entry of out is written by exactly one lane.
template <int SM_CH>
PK_DEVICE void relpos_bucket_sums(const float (&v)[SM_CH][8], float* __restrict__ out, int ld_r, int i, int mr, int n, int lane) {
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int k = 0; k < SM_CH; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int c = lane * 8 + k * 256 + e;
            if (c < n) {
                const int dist = c - i;
                if (dist <= -mr) lo += v[k][e];
                else if (dist >= mr) hi += v[k][e];
                else out[dist + mr] = v[k][e];
            }
        }
    lo = warp_sum(lo);
    hi = warp_sum(hi);
    for (int r = lane; r < ld_r; r += 32) {
        const int j = i - mr + r;
        if (r == 0) out[0] = lo;
        else if (r == 2 * mr) out[r] = hi;
        else if (r > 2 * mr || j < 0 || j >= n) out[r] = 0.f;
    }
}

// pk_softmax_masked_fwd with the key relations: S[r, j] + QR[rr, bucket(i, j)] is masked and normalised, and the bucket sums of
// the dropped-out probabilities Pd (as stored, i.e. rounded to T) go to Pb[rr, :].  rr = (sequence * q_len + i) * heads + head.
template <typename T, int SM_CH>
__global__ void __launch_bounds__(256) softmax_relpos_fwd_kernel(const float* __restrict__ S, long long ld_s, const float* __restrict__ QR,
                                                                 long long ld_r, T* __restrict__ P, T* __restrict__ Pd, long long ld_p,
                                                                 long long rows, int n, uint32_t drop_thresh, float drop_scale, uint32_t seed,
                                                                 int q_len, int heads, int causal, const uint8_t* __restrict__ key_pad,
                                                                 int mr, float* __restrict__ Pb) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        const long long seq = r / ((long long)heads * q_len);
        const int i = (int)(r % q_len), h = (int)((r / q_len) % heads);
        const long long rr = (seq * q_len + i) * heads + h;
        const float* sr = S + r * ld_s;
        const float* qr = QR + rr * ld_r;
        const int lim = causal ? min(n, i + 1) : n;
        const uint8_t* kp = key_pad ? key_pad + seq * n : nullptr;
        float v[SM_CH][8];
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) ld8f(sr + c0, v[k]);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int c = c0 + e;
                if (c >= lim || (kp && kp[c])) v[k][e] = -INFINITY;
                else v[k][e] += qr[relpos_bucket(c - i, mr)];
                mx = fmaxf(mx, v[k][e]);
            }
        }
        mx = warp_max(mx);
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < SM_CH; ++k)
#pragma unroll
            for (int e = 0; e < 8; ++e) { v[k][e] = __expf(v[k][e] - mx); s += v[k][e]; }
        const float inv = 1.f / warp_sum(s);
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) { o[e] = to_f32<T>(from_f32<T>(v[k][e] * inv)); v[k][e] = o[e]; }
                if (drop_thresh) {
                    const uint32_t salt = drop_row_salt((uint64_t)r, seed);
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const uint32_t km = drop_pair(salt, (uint32_t)((c0 >> 1) + e2), drop_thresh);
                        v[k][2 * e2] = (km & 1u) ? o[2 * e2] * drop_scale : 0.f;
                        v[k][2 * e2 + 1] = (km & 2u) ? o[2 * e2 + 1] * drop_scale : 0.f;
                    }
                }
                V8<T>::store(P + r * ld_p + c0, o);
                if (Pd != P) V8<T>::store(Pd + r * ld_p + c0, v[k]);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[k][e] = to_f32<T>(from_f32<T>(v[k][e]));
            }
        }
        relpos_bucket_sums<SM_CH>(v, Pb + rr * ld_r, (int)ld_r, i, mr, n, lane);
    }
}
// pk_softmax_bwd with the value relations: dPd[r, j] + G[rr, bucket(i, j)] (G = dO R^T) is the gradient of Pd; the bucket sums of
// dS (as stored) go to dSb[rr, :].
template <typename T, int SM_CH>
__global__ void __launch_bounds__(256) softmax_relpos_bwd_kernel(const float* __restrict__ dPd, long long ld_d, const float* __restrict__ G,
                                                                 long long ld_r, const T* __restrict__ P, long long ld_p, T* __restrict__ dS,
                                                                 long long rows, int n, uint32_t drop_thresh, float drop_scale, uint32_t seed,
                                                                 int q_len, int heads, int mr, float* __restrict__ dSb) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        const long long seq = r / ((long long)heads * q_len);
        const int i = (int)(r % q_len), h = (int)((r / q_len) % heads);
        const long long rr = (seq * q_len + i) * heads + h;
        const float* g = G + rr * ld_r;
        float d[SM_CH][8], pv[SM_CH][8];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
                ld8f(dPd + r * ld_d + c0, d[k]);
                V8<T>::load(P + r * ld_p + c0, pv[k]);
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    if (c0 + e < n) d[k][e] += g[relpos_bucket(c0 + e - i, mr)];
                if (drop_thresh) {
                    const uint32_t salt = drop_row_salt((uint64_t)r, seed);
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const uint32_t km = drop_pair(salt, (uint32_t)((c0 >> 1) + e2), drop_thresh);
                        d[k][2 * e2] = (km & 1u) ? d[k][2 * e2] * drop_scale : 0.f;
                        d[k][2 * e2 + 1] = (km & 2u) ? d[k][2 * e2 + 1] * drop_scale : 0.f;
                    }
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    if (c0 + e >= n) { d[k][e] = 0.f; pv[k][e] = 0.f; }
                    dot += d[k][e] * pv[k][e];
                }
            }
        }
        dot = warp_sum(dot);
#pragma unroll
        for (int k = 0; k < SM_CH; ++k) {
            const int c0 = lane * 8 + k * 256;
            if (c0 < (int)ld_p) {
#pragma unroll
                for (int e = 0; e < 8; ++e) d[k][e] = pv[k][e] * (d[k][e] - dot);
                V8<T>::store(dS + r * ld_p + c0, d[k]);
#pragma unroll
                for (int e = 0; e < 8; ++e) d[k][e] = to_f32<T>(from_f32<T>(d[k][e]));
            }
        }
        relpos_bucket_sums<SM_CH>(d, dSb + rr * ld_r, (int)ld_r, i, mr, n, lane);
    }
}

// =============================================================================== misc elementwise
// y = dropout(x) with the GEMM epilogue's index convention (flat index of a contiguous tensor); 8 elements per thread
// (scalar tail for n % 8), 16-byte accesses.
template <typename T>
__global__ void __launch_bounds__(256) dropout_kernel(const T* __restrict__ x, T* __restrict__ y, long long n, uint32_t thresh, float scale, uint32_t seed) {
    const long long nv = n / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
        float f[8];
        V8<T>::load(x + i * 8, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = drop_keep((uint64_t)(i * 8 + e), seed, thresh) ? f[e] * scale : 0.f;
        V8<T>::store(y + i * 8, f);
    }
    for (long long i = nv * 8 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = to_f32<T>(x[i]);
        y[i] = from_f32<T>(drop_keep((uint64_t)i, seed, thresh) ? v * scale : 0.f);
    }
}
// dx = dy * (y != 0) * scale     (backward of ReLU and of ReLU+dropout given the saved output y)
template <typename T>
__global__ void __launch_bounds__(256) mask_nz_kernel(const T* __restrict__ dy, const T* __restrict__ y, T* __restrict__ dx, long long n, float scale) {
    const long long nv = n / 8;
    constexpr int UR = 2;
    for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * UR; i0 < nv; i0 += (long long)gridDim.x * blockDim.x * UR) {
        float g[UR][8], f[UR][8];
#pragma unroll
        for (int k = 0; k < UR; ++k)
            if (i0 + k < nv) { V8<T>::load(dy + (i0 + k) * 8, g[k]); V8<T>::load(y + (i0 + k) * 8, f[k]); }
#pragma unroll
        for (int k = 0; k < UR; ++k)
            if (i0 + k < nv) {
#pragma unroll
                for (int e = 0; e < 8; ++e) g[k][e] = f[k][e] != 0.f ? g[k][e] * scale : 0.f;
                V8<T>::store(dx + (i0 + k) * 8, g[k]);
            }
    }
    for (long long i = nv * 8 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dx[i] = from_f32<T>(to_f32<T>(y[i]) != 0.f ? to_f32<T>(dy[i]) * scale : 0.f);
}
// out = a + b
template <typename T>
__global__ void __launch_bounds__(256) add_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ o, long long n) {
    const long long nv = n / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
        float f[8], g[8];
        V8<T>::load(a + i * 8, f);
        V8<T>::load(b + i * 8, g);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] += g[e];
        V8<T>::store(o + i * 8, f);
    }
    for (long long i = nv * 8 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        o[i] = from_f32<T>(to_f32<T>(a[i]) + to_f32<T>(b[i]));
}
// log_softmax rows: x T [rows, ld] (first n valid) -> y f32 [rows, n] * 1
template <typename T>
__global__ void __launch_bounds__(256) log_softmax_kernel(const T* __restrict__ x, long long ld, float* __restrict__ y, long long rows,
                                                          int n, float scale, float* __restrict__ lse = nullptr) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        const T* xr = x + r * ld;
        float m = -INFINITY;
        for (int c = lane; c < n; c += 32) m = fmaxf(m, to_f32<T>(xr[c]) * scale);
        m = warp_max(m);
        float s = 0.f;
        for (int c = lane; c < n; c += 32) s += expf(to_f32<T>(xr[c]) * scale - m);
        const float l = m + logf(warp_sum(s));
        if (y) for (int c = lane; c < n; c += 32) y[r * n + c] = to_f32<T>(xr[c]) * scale - l;
        if (lse && lane == 0) lse[r] = l;                          // y[r, c] == x[r, c] * scale - lse[r], bit for bit (same expression)
    }
}

// =============================================================================== gated joint
// h[b,t,u,c] = tanh(e1[b,t,c] + p1[b,u,c]) * sigmoid(eg[b,t,c] + pg[b,u,c])
// ex = [B*T, 2H] (cols [0,H) = fc1 part, [H,2H) = gate part), py = [B*U1, 2H]; biases already folded into ex.
PK_DEVICE float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
// the activation pair jt_tanh / jt_sigmoid lives in common.cuh (shared with the pruned joint, rnnt_pruned.cu)

template <typename T>
__global__ void __launch_bounds__(128) joint_gate_fwd_kernel(const T* __restrict__ ex, const T* __restrict__ py, T* __restrict__ h,
                                                             int B, int Tt, int U1, int H, int ld_h) {
    // one CTA per (b,t); threads over channels (8 each); loop over u.  When ld_h > H the 8 pad columns hold
    // (1, 0, ..., 0): the ones column turns the fc2 bias gradient into one extra column of the wgrad GEMM.
    const int bt = blockIdx.x;
    const int b = bt / Tt;
    for (int c0 = threadIdx.x * 8; c0 < H; c0 += blockDim.x * 8) {
        float e1[8], eg[8];
        V8<T>::load(ex + (long long)bt * 2 * H + c0, e1);
        V8<T>::load(ex + (long long)bt * 2 * H + H + c0, eg);
        for (int u = 0; u < U1; ++u) {
            float p1[8], pg[8], o[8];
            const T* pr = py + ((long long)b * U1 + u) * 2 * H;
            V8<T>::load(pr + c0, p1);
            V8<T>::load(pr + H + c0, pg);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = jt_tanh<T>(e1[e] + p1[e]) * jt_sigmoid<T>(eg[e] + pg[e]);
            V8<T>::store(h + ((long long)bt * U1 + u) * ld_h + c0, o);
        }
    }
    if (ld_h > H) {
        for (int u = threadIdx.x; u < U1; u += blockDim.x) {
            const float one[8] = {1.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            V8<T>::store(h + ((long long)bt * U1 + u) * ld_h + H, one);
        }
    }
}
// forward, channel-sliced form: one CTA per (batch element, 32-channel slice) keeps its slice of py (all labels) in shared memory and
// walks the frames, so py is read from L2 once per slice instead of once per (b, t) CTA (the frame-major kernel above re-reads the
// whole [U1, 2H] block of its utterance for every frame: 4.7 GB of L2 reads at the config-2 shape, more than the 2.4 GB it writes).
// Lanes: 4 channel groups x 8 labels per warp (a warp's store covers 64 contiguous bytes of 8 rows), 4 warps = 32 labels per pass.
template <typename T, int UI>
__global__ void __launch_bounds__(128) joint_gate_fwd_sliced_kernel(const T* __restrict__ ex, const T* __restrict__ py, T* __restrict__ h,
                                                                    int B, int Tt, int U1, int H, int ld_h) {
    extern __shared__ __align__(16) uint8_t jg_smem[];
    T* s_py = reinterpret_cast<T*>(jg_smem);                   // [2 parts][4 channel groups][U1][8]
    const int slices = H / 32;
    const int b = blockIdx.x / slices, cs = blockIdx.x - b * slices;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ct = lane & 3, ul = (lane >> 2) + 8 * warp;
    const int c0 = cs * 32 + ct * 8;
    for (int i = tid; i < U1 * 8; i += 128) {
        const int u = i >> 3, v = i & 7;
        float f[8];
        V8<T>::load(py + ((long long)b * U1 + u) * 2 * H + (v >> 2) * H + cs * 32 + (v & 3) * 8, f);
        V8<T>::store(s_py + ((long long)(v * U1) + u) * 8, f);
    }
    __syncthreads();
    const T* s_p1 = s_py + (long long)(ct * U1) * 8;
    const T* s_pg = s_py + (long long)((4 + ct) * U1) * 8;
    const T* ex_b = ex + (long long)b * Tt * 2 * H + c0;
    typename V8<T>::Raw e1n = V8<T>::load_raw(ex_b), egn = V8<T>::load_raw(ex_b + H);
    for (int t = 0; t < Tt; ++t) {
        float e1[8], eg[8];
        V8<T>::unpack(e1n, e1);
        V8<T>::unpack(egn, eg);
        if (t + 1 < Tt) {
            e1n = V8<T>::load_raw(ex_b + (long long)(t + 1) * 2 * H);
            egn = V8<T>::load_raw(ex_b + (long long)(t + 1) * 2 * H + H);
        }
        T* hrow = h + ((long long)(b * Tt + t) * U1) * ld_h + c0;
#pragma unroll
        for (int i = 0; i < UI; ++i) {
            const int u = ul + 32 * i;
            if (u < U1) {
                float p1[8], pg[8], o[8];
                V8<T>::load(s_p1 + u * 8, p1);
                V8<T>::load(s_pg + u * 8, pg);
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = jt_tanh<T>(e1[e] + p1[e]) * jt_sigmoid<T>(eg[e] + pg[e]);
                V8<T>::store(hrow + (long long)u * ld_h, o);
            }
        }
        if (ld_h > H && cs == 0 && ct == 0) {                   // the ones column of the fc2 bias gradient (see the frame-major kernel)
            const float one[8] = {1.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < UI; ++i) {
                const int u = ul + 32 * i;
                if (u < U1) V8<T>::store(h + ((long long)(b * Tt + t) * U1 + u) * ld_h + H, one);
            }
        }
    }
}
// dh row of joint row r: dh[r], or with a row map (compacted joint gradient, pk_rnnt_loss_fwd_bwd_compact) dh[map[r]], zeros when
// map[r] < 0.  A zero row adds +-0 to every sum below, so the sums equal the dense ones apart from the sign of a zero.
template <typename T> PK_DEVICE typename V8<T>::Raw load_dh_mapped(const T* dh, int m, int H, int c0) {
    if (m >= 0) return V8<T>::load_raw(dh + (long long)m * H + c0);
    return typename V8<T>::Raw{};
}
template <typename T> PK_DEVICE typename V8<T>::Raw load_dh_row(const T* dh, const int* map, long long r, int H, int c0) {
    if (map == nullptr) return V8<T>::load_raw(dh + r * H + c0);
    return load_dh_mapped<T>(dh, __ldg(map + r), H, c0);
}

// backward, reduction over u:  dex[b,t,:] = sum_u (d1, dg);    d1 = dh*g*(1-a^2), dg = dh*a*g*(1-g)
template <typename T>
__global__ void __launch_bounds__(128) joint_gate_bwd_ex_kernel(const T* __restrict__ ex, const T* __restrict__ py,
                                                                const T* __restrict__ dh, const int* __restrict__ dh_map,
                                                                T* __restrict__ dex, int B, int Tt, int U1, int H) {
    const int bt = blockIdx.x;
    const int b = bt / Tt;
    for (int c0 = threadIdx.x * 8; c0 < H; c0 += blockDim.x * 8) {
        float e1[8], eg[8], a1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ag[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        V8<T>::load(ex + (long long)bt * 2 * H + c0, e1);
        V8<T>::load(ex + (long long)bt * 2 * H + H + c0, eg);
        for (int u = 0; u < U1; ++u) {
            float p1[8], pg[8], d[8];
            const T* pr = py + ((long long)b * U1 + u) * 2 * H;
            V8<T>::load(pr + c0, p1);
            V8<T>::load(pr + H + c0, pg);
            V8<T>::unpack(load_dh_row<T>(dh, dh_map, (long long)bt * U1 + u, H, c0), d);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float a = jt_tanh<T>(e1[e] + p1[e]), g = jt_sigmoid<T>(eg[e] + pg[e]);
                a1[e] += d[e] * g * (1.f - a * a);
                ag[e] += d[e] * a * g * (1.f - g);
            }
        }
        V8<T>::store(dex + (long long)bt * 2 * H + c0, a1);
        V8<T>::store(dex + (long long)bt * 2 * H + H + c0, ag);
    }
}
// backward, reduction over t: one CTA per (b,u)
template <typename T>
__global__ void __launch_bounds__(128) joint_gate_bwd_py_kernel(const T* __restrict__ ex, const T* __restrict__ py,
                                                                const T* __restrict__ dh, const int* __restrict__ dh_map,
                                                                T* __restrict__ dpy, int B, int Tt, int U1, int H) {
    const int bu = blockIdx.x;
    const int b = bu / U1, u = bu - b * U1;
    for (int c0 = threadIdx.x * 8; c0 < H; c0 += blockDim.x * 8) {
        float p1[8], pg[8], a1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ag[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        V8<T>::load(py + (long long)bu * 2 * H + c0, p1);
        V8<T>::load(py + (long long)bu * 2 * H + H + c0, pg);
        for (int t = 0; t < Tt; ++t) {
            float e1[8], eg[8], d[8];
            const long long bt = (long long)b * Tt + t;
            V8<T>::load(ex + bt * 2 * H + c0, e1);
            V8<T>::load(ex + bt * 2 * H + H + c0, eg);
            V8<T>::unpack(load_dh_row<T>(dh, dh_map, bt * U1 + u, H, c0), d);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float a = jt_tanh<T>(e1[e] + p1[e]), g = jt_sigmoid<T>(eg[e] + pg[e]);
                a1[e] += d[e] * g * (1.f - a * a);
                ag[e] += d[e] * a * g * (1.f - g);
            }
        }
        V8<T>::store(dpy + (long long)bu * 2 * H + c0, a1);
        V8<T>::store(dpy + (long long)bu * 2 * H + H + c0, ag);
    }
}

// backward, BOTH reductions in one pass over dh: one CTA per (batch element, 32-channel slice), one WARP per 8 channels, the 32
// lanes of a warp over the labels: a lane owns u = lane + 32 i (i < UI) of its warp's 8 channels for ALL frames, so its dpy sums stay
// in registers for the whole kernel (the sum over t runs in one thread, in frame order, like the two-pass kernel), while the dex sums
// of a frame are reduced over the lanes by a transposing butterfly (16 values over 32 lanes in 16 shuffles).  Warps never meet after
// the prologue.  dh is read once (the two-pass form read it twice) and every tanh / sigmoid is evaluated once instead of twice.
template <typename T, int UI>
__global__ void __launch_bounds__(128) joint_gate_bwd_fused_kernel(const T* __restrict__ ex, const T* __restrict__ py, const T* __restrict__ dh,
                                                                   const int* __restrict__ dh_map, T* __restrict__ dex, T* __restrict__ dpy,
                                                                   int B, int Tt, int U1, int H) {
    extern __shared__ __align__(16) uint8_t jg_smem[];
    T* s_py = reinterpret_cast<T*>(jg_smem);                   // [2 parts][4 channel groups][U1][8]: conflict-free 16-byte rows per lane
    const int slices = H / 32;
    const int b = blockIdx.x / slices, cs = blockIdx.x - b * slices;
    const int tid = threadIdx.x, ct = tid >> 5, lane = tid & 31;
    const int c0 = cs * 32 + ct * 8;
    for (int i = tid; i < U1 * 8; i += 128) {
        const int u = i >> 3, v = i & 7;                       // v < 4: fc1 part, else gate part; v & 3 = channel group
        float f[8];
        V8<T>::load(py + ((long long)b * U1 + u) * 2 * H + (v >> 2) * H + cs * 32 + (v & 3) * 8, f);
        V8<T>::store(s_py + ((long long)(v * U1) + u) * 8, f);
    }
    float a1u[UI][8], agu[UI][8];
#pragma unroll
    for (int i = 0; i < UI; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) { a1u[i][e] = 0.f; agu[i][e] = 0.f; }
    __syncthreads();
    const T* s_p1 = s_py + (long long)(ct * U1) * 8;
    const T* s_pg = s_py + (long long)((4 + ct) * U1) * 8;
    const long long row_b = (long long)b * Tt * U1;            // joint row of (b, 0, 0)
    const T* ex_b = ex + (long long)b * Tt * 2 * H + c0;
    typename V8<T>::Raw dn[UI], e1n, egn;                      // next frame's operands, fetched one frame ahead (kept packed)
    int mn[UI];                                                // with a row map: its entries for the frame after next
#pragma unroll
    for (int i = 0; i < UI; ++i) {
        const int u = lane + 32 * i;
        if (u < U1) dn[i] = load_dh_row<T>(dh, dh_map, row_b + u, H, c0);
        mn[i] = (dh_map != nullptr && u < U1 && Tt > 1) ? __ldg(dh_map + row_b + U1 + u) : -1;
    }
    e1n = V8<T>::load_raw(ex_b);
    egn = V8<T>::load_raw(ex_b + H);
    for (int t = 0; t < Tt; ++t) {
        float e1[8], eg[8];
        typename V8<T>::Raw dc[UI];
        V8<T>::unpack(e1n, e1);
        V8<T>::unpack(egn, eg);
#pragma unroll
        for (int i = 0; i < UI; ++i) dc[i] = dn[i];
        if (t + 1 < Tt) {
#pragma unroll
            for (int i = 0; i < UI; ++i) {
                const int u = lane + 32 * i;
                if (u < U1) {
                    if (dh_map == nullptr) {
                        dn[i] = V8<T>::load_raw(dh + (row_b + (long long)(t + 1) * U1 + u) * H + c0);
                    } else {                                   // the map entry came one frame earlier: no dependent load here
                        dn[i] = load_dh_mapped<T>(dh, mn[i], H, c0);
                        if (t + 2 < Tt) mn[i] = __ldg(dh_map + row_b + (long long)(t + 2) * U1 + u);
                    }
                }
            }
            e1n = V8<T>::load_raw(ex_b + (long long)(t + 1) * 2 * H);
            egn = V8<T>::load_raw(ex_b + (long long)(t + 1) * 2 * H + H);
        }
        float v[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) v[e] = 0.f;
#pragma unroll
        for (int i = 0; i < UI; ++i) {
            const int u = lane + 32 * i;
            if (u < U1) {
                float p1[8], pg[8], d[8];
                V8<T>::unpack(dc[i], d);
                V8<T>::load(s_p1 + u * 8, p1);
                V8<T>::load(s_pg + u * 8, pg);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float a = jt_tanh<T>(e1[e] + p1[e]), g = jt_sigmoid<T>(eg[e] + pg[e]);
                    const float dg = d[e] * g;
                    const float t1 = dg * (1.f - a * a), tg = dg * a * (1.f - g);
                    a1u[i][e] += t1; agu[i][e] += tg;
                    v[e] += t1; v[8 + e] += tg;
                }
            }
        }
        // 16 sums x 32 lanes -> lane l ends with sum number (l >> 1)
        float w8[8], w4[4], w2[2];
        const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4, h2 = lane & 2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float keep = h16 ? v[i + 8] : v[i], send = h16 ? v[i] : v[i + 8];
            w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float keep = h8 ? w8[i + 4] : w8[i], send = h8 ? w8[i] : w8[i + 4];
            w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float keep = h4 ? w4[i + 2] : w4[i], send = h4 ? w4[i] : w4[i + 2];
            w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
        float w1 = (h2 ? w2[1] : w2[0]) + __shfl_xor_sync(0xffffffffu, h2 ? w2[0] : w2[1], 2);
        w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
        if ((lane & 1) == 0) {
            const int j = lane >> 1;                           // = 8*h16 + 4*h8 + 2*h4 + h2: fc1 sums 0..7, gate sums 8..15
            dex[((long long)b * Tt + t) * 2 * H + (j >> 3) * H + c0 + (j & 7)] = from_f32<T>(w1);
        }
    }
#pragma unroll
    for (int i = 0; i < UI; ++i) {
        const int u = lane + 32 * i;
        if (u < U1) {
            V8<T>::store(dpy + ((long long)b * U1 + u) * 2 * H + c0, a1u[i]);
            V8<T>::store(dpy + ((long long)b * U1 + u) * 2 * H + H + c0, agu[i]);
        }
    }
}

// =============================================================================== LSTM cell (gate order i,f,g,o)
// gates = gx[b, :4H] + gh[b, :4H] (f32 both: gx holds W_ih x + b_ih + b_hh for this step)
template <typename T>
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ gx, long long ld_gx, const float* __restrict__ gh, long long ld_gh,
                                     const float* __restrict__ c_prev, float* __restrict__ c_out, T* __restrict__ h_out,
                                     long long ld_h, float* __restrict__ gates_save, int B, int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* a = gx + (long long)b * ld_gx;
    float gi = a[j], gf = a[H + j], gg = a[2 * H + j], go = a[3 * H + j];
    if (gh) {
        const float* r = gh + (long long)b * ld_gh;
        gi += r[j]; gf += r[H + j]; gg += r[2 * H + j]; go += r[3 * H + j];
    }
    gi = sigmoidf_(gi); gf = sigmoidf_(gf); gg = tanhf(gg); go = sigmoidf_(go);
    const float cp = c_prev ? c_prev[i] : 0.f;
    const float c = gf * cp + gi * gg;
    c_out[i] = c;
    h_out[(long long)b * ld_h + j] = from_f32<T>(go * tanhf(c));
    if (gates_save) {
        float* g = gates_save + (long long)b * 4 * H;
        g[j] = gi; g[H + j] = gf; g[2 * H + j] = gg; g[3 * H + j] = go;
    }
}
// dh_total = dh_out(t) + dh_rec; produces d(pre-activation gates) as T [B,4H] and dc_prev
template <typename T>
__global__ void lstm_cell_bwd_kernel(const T* __restrict__ dh_out, long long ld_dho, const float* __restrict__ dh_rec,
                                     const float* __restrict__ dc_next, const float* __restrict__ gates, const float* __restrict__ c,
                                     const float* __restrict__ c_prev, T* __restrict__ dgates, float* __restrict__ dc_prev, int B,
                                     int H) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H) return;
    const int b = i / H, j = i - b * H;
    const float* g = gates + (long long)b * 4 * H;
    const float gi = g[j], gf = g[H + j], gg = g[2 * H + j], go = g[3 * H + j];
    float dh = dh_out ? to_f32<T>(dh_out[(long long)b * ld_dho + j]) : 0.f;
    if (dh_rec) dh += dh_rec[i];
    const float tc = tanhf(c[i]);
    float dc = dh * go * (1.f - tc * tc);
    if (dc_next) dc += dc_next[i];
    const float cp = c_prev ? c_prev[i] : 0.f;
    T* d = dgates + (long long)b * 4 * H;
    d[j] = from_f32<T>(dc * gg * gi * (1.f - gi));
    d[H + j] = from_f32<T>(dc * cp * gf * (1.f - gf));
    d[2 * H + j] = from_f32<T>(dc * gi * (1.f - gg * gg));
    d[3 * H + j] = from_f32<T>(dh * tc * go * (1.f - go));
    dc_prev[i] = dc * gf;
}

// =============================================================================== embedding
template <typename T>
__global__ void embedding_fwd_kernel(const long long* __restrict__ idx, const float* __restrict__ table, int E, T* __restrict__ out,
                                     int ld_out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n * ld_out; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / ld_out;
        const int c = (int)(i - r * ld_out);
        out[i] = from_f32<T>(c < E ? table[idx[r] * E + c] : 0.f);
    }
}
template <typename T>
__global__ void embedding_bwd_kernel(const long long* __restrict__ idx, const T* __restrict__ dout, int ld, int E,
                                     float* __restrict__ dtable, long long n, long long padding_idx) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n * E; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / E;
        const int c = (int)(i - r * E);
        if (idx[r] != padding_idx) atomicAdd(&dtable[idx[r] * E + c], to_f32<T>(dout[r * ld + c]));
    }
}


// =============================================================================== MBR path helpers
// dst[r, :] = src[idx[r], :]
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ src, const int* __restrict__ idx, T* __restrict__ dst, long long rows, int C) {
    const long long r = blockIdx.x;
    if (r >= rows) return;
    const T* s = src + (long long)idx[r] * C;
    for (int c = threadIdx.x * 8; c < C; c += blockDim.x * 8) {
        float f[8];
        V8<T>::load(s + c, f);
        V8<T>::store(dst + r * C + c, f);
    }
}
// dst[idx[r], :] += src[r, :]   (f32 accumulation)
template <typename T>
__global__ void scatter_add_rows_kernel(const T* __restrict__ src, const int* __restrict__ idx, float* __restrict__ dst, long long rows, int C) {
    const long long r = blockIdx.x;
    if (r >= rows) return;
    float* d = dst + (long long)idx[r] * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&d[c], to_f32<T>(src[r * C + c]));
}
// gradient of sum_r coef[r] * log_softmax(scale * z[r])[tok[r]] w.r.t. z:  scale * coef * (onehot - softmax(scale z))
template <typename T>
__global__ void __launch_bounds__(256) ce_grad_kernel(const T* __restrict__ z, long long ld, const int* __restrict__ tok,
                                                      const float* __restrict__ coef, float scale, T* __restrict__ dz, long long rows, int n) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = warp; r < rows; r += nw) {
        const T* zr = z + r * ld;
        T* dr = dz + r * ld;
        const float cf = coef[r];
        if (cf == 0.f) {
            for (int c = lane; c < (int)ld; c += 32) dr[c] = from_f32<T>(0.f);
            continue;
        }
        float m = -INFINITY;
        for (int c = lane; c < n; c += 32) m = fmaxf(m, to_f32<T>(zr[c]) * scale);
        m = warp_max(m);
        float sum = 0.f;
        for (int c = lane; c < n; c += 32) sum += expf(to_f32<T>(zr[c]) * scale - m);
        const float inv = 1.f / warp_sum(sum);
        const int y = tok[r];
        for (int c = lane; c < (int)ld; c += 32) {
            float g = 0.f;
            if (c < n) g = scale * cf * ((c == y ? 1.f : 0.f) - expf(to_f32<T>(zr[c]) * scale - m) * inv);
            dr[c] = from_f32<T>(g);
        }
    }
}
}  // namespace pk

// ================================================================================================ C ABI
using namespace pk;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define DONE() PK_CHECK_LAUNCH(); count_launch(); return 0

// column statistics in two deterministic stages; ws must hold pk_colstats_ws_floats(C) floats
static const int kColGy = 296;
extern "C" long long pk_colstats_ws_floats(int C) { return (long long)kColGy * 2 * C; }
template <typename T, int MODE>
static int run_colstats(const T* x, const T* aux, long long rows, int C, const float* mean, const float* rstd, float* ws, float* out1,
                        float* out2, cudaStream_t st) {
    int gy = (int)((rows + 63) / 64);
    if (gy > kColGy) gy = kColGy;
    if (gy < 1) gy = 1;
    dim3 g((C / 8 + 127) / 128, gy);
    colstats_kernel<T, MODE><<<g, 128, 0, st>>>(x, aux, rows, C, mean, rstd, ws);
    PK_CHECK_LAUNCH(); count_launch();
    colstats_reduce_kernel<<<(C + 31) / 32, 256, 0, st>>>(ws, gy, C, out1, out2);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

static uint32_t drop_thresh_of(float p) {
    if (p <= 0.f) return 0u;
    double t = (double)p * 4294967296.0;
    uint32_t r = t >= 4294967295.0 ? 4294967295u : (uint32_t)t;
    return r == 0 ? 1u : r;
}

extern "C" int pk_cast_split(const void* src, int src_dtype, long long ld_src, void* hi, void* lo, long long ld_dst,
                             long long rows, int cols, int cols_pad, float scale, void* stream) {
    PK_CHECK_ARG(rows > 0 && cols > 0 && cols_pad >= cols, "bad shape");
    const int grid = grid_for(rows * cols_pad, 256);
    if (src_dtype == PK_F32)
        cast_split_kernel<float><<<grid, 256, 0, STREAM(stream)>>>((const float*)src, ld_src, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo,
                                                                  ld_dst, rows, cols, cols_pad, scale);
    else
        cast_split_kernel<__nv_bfloat16><<<grid, 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)src, ld_src, (__nv_bfloat16*)hi,
                                                                          (__nv_bfloat16*)lo, ld_dst, rows, cols, cols_pad, scale);
    DONE();
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

/* BatchNorm1d over rows of x [rows, C].  stats_ws: pk_colstats_ws_floats(C) + 2*C floats of scratch. */
extern "C" int pk_bn_fwd(const void* x, void* y, int dtype, long long rows, int C, const float* w, const float* b, float eps,
                         int train, float momentum, float* run_mean, float* run_var, float* mean, float* rstd, float* stats_ws,
                         void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0, "C must be a multiple of 8 and rows > 0");
    PK_CHECK_ARG(aligned16(x) && aligned16(y) && (!train || aligned16(stats_ws)), "pk_bn_fwd: x, y, stats_ws must be 16-byte aligned");
    cudaStream_t st = STREAM(stream);
    if (train) {
        float* sums = stats_ws + pk_colstats_ws_floats(C);
        PK_DISPATCH_T(dtype, {
            int rc = run_colstats<T, 2>((const T*)x, nullptr, rows, C, nullptr, nullptr, stats_ws, sums, sums + C, st);
            if (rc) return rc;
            bn_finalize_kernel<T><<<(C + 255) / 256, 256, 0, st>>>((const T*)x, sums, sums + C, rows, C, eps, momentum, mean, rstd, run_mean,
                                                                 run_var);
        });
    } else {
        bn_eval_stats_kernel<<<(C + 255) / 256, 256, 0, st>>>(run_mean, run_var, C, eps, mean, rstd);
    }
    PK_CHECK_LAUNCH(); count_launch();
    PK_DISPATCH_T(dtype, (bn_apply_kernel<T><<<col_grid(rows, C), 128, 0, st>>>((const T*)x, (T*)y, rows, C, mean, rstd, w, b)));
    DONE();
}

/* dx (optionally ReLU-masked by x > 0), dw[C], db[C] (overwritten).  stats_ws: 2*C floats. */
extern "C" int pk_bn_bwd(const void* dy, const void* x, void* dx, int dtype, long long rows, int C, const float* w,
                         const float* mean, const float* rstd, int train, int relu_mask, float* dw, float* db, float* ws,
                         void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0, "C must be a multiple of 8 and rows > 0");
    PK_CHECK_ARG(aligned16(dy) && aligned16(x) && aligned16(dx) && aligned16(ws), "pk_bn_bwd: dy, x, dx, ws must be 16-byte aligned");
    cudaStream_t st = STREAM(stream);
    PK_DISPATCH_T(dtype, { int rc = run_colstats<T, 1>((const T*)dy, (const T*)x, rows, C, mean, rstd, ws, db, dw, st); if (rc) return rc; });
    PK_DISPATCH_T(dtype, (bn_bwd_apply_kernel<T><<<col_grid(rows, C), 128, 0, st>>>((const T*)dy, (const T*)x, (T*)dx, rows, C, mean, rstd, w,
                                                                       train ? db : nullptr, train ? dw : nullptr, relu_mask)));
    DONE();
}

extern "C" int pk_colsum(const void* x, int dtype, long long rows, int C, float* out, float* ws, void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0, "C must be a multiple of 8 and rows > 0");
    PK_CHECK_ARG(aligned16(x) && aligned16(ws), "pk_colsum: x, ws must be 16-byte aligned");
    cudaStream_t st = STREAM(stream);
    PK_DISPATCH_T(dtype, { int rc = run_colstats<T, 0>((const T*)x, nullptr, rows, C, nullptr, nullptr, ws, out, nullptr, st); if (rc) return rc; });
    return 0;
}

extern "C" int pk_layernorm_fwd(const void* x, void* y, int dtype, long long rows, int C, const float* w, const float* b, float eps,
                                float* mean, float* rstd, void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0 && C <= 1024, "C must be a multiple of 8, <= 1024, and rows > 0");
    PK_CHECK_ARG(aligned16(x) && aligned16(y), "pk_layernorm_fwd: x, y must be 16-byte aligned");
    const int grid = grid_for(rows, 8);
    PK_DISPATCH_T(dtype, (ln_fwd_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)x, (T*)y, rows, C, w, b, eps, mean, rstd)));
    DONE();
}
extern "C" int pk_layernorm_bwd(const void* dy, const void* x, void* dx, int dtype, long long rows, int C, const float* w,
                                const float* mean, const float* rstd, float* dw, float* db, void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0 && C <= 1024, "C must be a multiple of 8, <= 1024, and rows > 0");
    PK_CHECK_ARG(aligned16(dy) && aligned16(x) && aligned16(dx), "pk_layernorm_bwd: dy, x, dx must be 16-byte aligned");
    cudaStream_t st = STREAM(stream);
    PK_CHECK_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * C, st));
    PK_CHECK_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * C, st));
    const int grid = grid_for(rows, 8, 2);
    PK_DISPATCH_T(dtype, (ln_bwd_kernel<T><<<grid, 256, 2 * C * sizeof(float), st>>>((const T*)dy, (const T*)x, (T*)dx, rows, C, w, mean,
                                                                                     rstd, dw, db)));
    DONE();
}

extern "C" int pk_softmax_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                              float drop_p, uint32_t seed, void* stream) {
    PK_CHECK_ARG(rows > 0 && n > 0 && ld_p >= n && ld_s >= ld_p && ld_p <= 2048 && ld_p % 8 == 0 && ld_s % 8 == 0, "softmax rows: ld % 8 == 0, <= 2048 wide");
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);     // 16-bit pair mask (common.cuh drop_pair)
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 4><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed))); }
    else { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 8><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed))); }
    DONE();
}
extern "C" int pk_softmax_masked_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                                     int q_len, int heads, int causal, const uint8_t* key_pad, float drop_p, uint32_t seed, void* stream) {
    PK_CHECK_ARG(rows > 0 && n > 0 && ld_p >= n && ld_s >= ld_p && ld_p <= 2048 && ld_p % 8 == 0 && ld_s % 8 == 0, "softmax rows: ld % 8 == 0, <= 2048 wide");
    PK_CHECK_ARG(q_len > 0 && heads > 0 && rows % ((long long)heads * q_len) == 0, "masked softmax: rows = sequences * heads * q_len");
    PK_CHECK_ARG(causal || key_pad, "masked softmax without a mask: use pk_softmax_fwd");
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 4><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, q_len, heads, causal, key_pad))); }
    else { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 8><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, q_len, heads, causal, key_pad))); }
    DONE();
}
extern "C" int pk_softmax_chunk_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                                    int chunk_len, int chunk_off, int left_chunks, float drop_p, uint32_t seed, void* stream) {
    PK_CHECK_ARG(rows > 0 && n > 0 && ld_p >= n && ld_s >= ld_p && ld_p <= 2048 && ld_p % 8 == 0 && ld_s % 8 == 0, "softmax rows: ld % 8 == 0, <= 2048 wide");
    PK_CHECK_ARG(rows % n == 0, "chunked softmax: rows = sequences * heads * n");
    PK_CHECK_ARG(chunk_len >= 1 && chunk_off >= 0 && left_chunks >= -1, "chunk mask: chunk_len >= 1, chunk_off >= 0, left_chunks >= -1");
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 4, true><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, n, 1, 0, nullptr, chunk_len, chunk_off, left_chunks))); }
    else { PK_DISPATCH_T(dtype, (softmax_fwd_kernel<T, 8, true><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, n, 1, 0, nullptr, chunk_len, chunk_off, left_chunks))); }
    DONE();
}
extern "C" int pk_softmax_bwd(const float* dPd, long long ld_d, const void* P, long long ld_p, void* dS, int dtype, long long rows,
                              int n, float drop_p, uint32_t seed, void* stream) {
    PK_CHECK_ARG(rows > 0 && n > 0 && ld_p >= n && ld_d >= ld_p && ld_p <= 2048 && ld_p % 8 == 0 && ld_d % 8 == 0, "softmax rows: ld % 8 == 0, <= 2048 wide");
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);     // 16-bit pair mask (common.cuh drop_pair)
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_bwd_kernel<T, 4><<<grid, 256, 0, STREAM(stream)>>>(dPd, ld_d, (const T*)P, ld_p, (T*)dS, rows, n, th, sc, seed))); }
    else { PK_DISPATCH_T(dtype, (softmax_bwd_kernel<T, 8><<<grid, 256, 0, STREAM(stream)>>>(dPd, ld_d, (const T*)P, ld_p, (T*)dS, rows, n, th, sc, seed))); }
    DONE();
}
#define PK_RELPOS_CHECKS(ld_x, ld_p)                                                                                                  \
    PK_CHECK_ARG(rows > 0 && n > 0 && ld_p >= n && ld_x >= ld_p && ld_p <= 2048 && ld_p % 8 == 0 && ld_x % 8 == 0,                     \
                 "relative-position softmax rows: n <= ld_p <= 2048, pitches multiples of 8");                                         \
    PK_CHECK_ARG(q_len == n && heads > 0 && rows % ((long long)heads * q_len) == 0,                                                     \
                 "relative-position softmax: self-attention rows = sequences * heads * n");                                             \
    PK_CHECK_ARG(max_rel >= 1 && max_rel <= PK_RELPOS_MAX && ld_r >= 2 * max_rel + 1 && ld_r % 8 == 0,                               \
                 "relative positions: 1 <= max_rel <= 1024, ld_r >= 2*max_rel + 1 and a multiple of 8")
extern "C" int pk_softmax_masked_relpos_fwd(const float* S, long long ld_s, const float* QR, long long ld_r, void* P, void* Pd, int dtype,
                                            long long ld_p, long long rows, int n, int q_len, int heads, int causal, const uint8_t* key_pad,
                                            int max_rel, float* Pb, float drop_p, uint32_t seed, void* stream) {
    PK_RELPOS_CHECKS(ld_s, ld_p);
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_relpos_fwd_kernel<T, 4><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, QR, ld_r, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, q_len, heads, causal, key_pad, max_rel, Pb))); }
    else { PK_DISPATCH_T(dtype, (softmax_relpos_fwd_kernel<T, 8><<<grid, 256, 0, STREAM(stream)>>>(S, ld_s, QR, ld_r, (T*)P, (T*)Pd, ld_p, rows, n, th, sc, seed, q_len, heads, causal, key_pad, max_rel, Pb))); }
    DONE();
}
extern "C" int pk_softmax_relpos_bwd(const float* dPd, long long ld_d, const float* G, long long ld_r, const void* P, long long ld_p, void* dS,
                                     int dtype, long long rows, int n, int q_len, int heads, int max_rel, float* dSb, float drop_p,
                                     uint32_t seed, void* stream) {
    PK_RELPOS_CHECKS(ld_d, ld_p);
    const int grid = grid_for(rows, 8);
    const uint32_t th = drop_thresh16_of(drop_p);
    const float sc = drop_scale16_of(th);
    if (ld_p <= 1024) { PK_DISPATCH_T(dtype, (softmax_relpos_bwd_kernel<T, 4><<<grid, 256, 0, STREAM(stream)>>>(dPd, ld_d, G, ld_r, (const T*)P, ld_p, (T*)dS, rows, n, th, sc, seed, q_len, heads, max_rel, dSb))); }
    else { PK_DISPATCH_T(dtype, (softmax_relpos_bwd_kernel<T, 8><<<grid, 256, 0, STREAM(stream)>>>(dPd, ld_d, G, ld_r, (const T*)P, ld_p, (T*)dS, rows, n, th, sc, seed, q_len, heads, max_rel, dSb))); }
    DONE();
}
#undef PK_RELPOS_CHECKS

extern "C" int pk_dropout(const void* x, void* y, int dtype, long long n, float p, uint32_t seed, void* stream) {
    const int grid = grid_for(n, 256 * 8);
    const uint32_t th = drop_thresh_of(p);
    PK_CHECK_ARG(th != 0, "p must be > 0");
    PK_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "pk_dropout: pointers must be 16-byte aligned");
    PK_DISPATCH_T(dtype, (dropout_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)x, (T*)y, n, th, 1.f / (1.f - p), seed)));
    DONE();
}
extern "C" int pk_mask_nz(const void* dy, const void* y, void* dx, int dtype, long long n, float scale, void* stream) {
    const int grid = grid_for(n, 256 * 16);
    PK_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0, "pk_mask_nz: pointers must be 16-byte aligned");
    PK_DISPATCH_T(dtype, (mask_nz_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)dy, (const T*)y, (T*)dx, n, scale)));
    DONE();
}
extern "C" int pk_add(const void* a, const void* b, void* o, int dtype, long long n, void* stream) {
    const int grid = grid_for(n, 256 * 8);
    PK_CHECK_ARG(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(o)) & 15) == 0, "pk_add: pointers must be 16-byte aligned");
    PK_DISPATCH_T(dtype, (add_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)a, (const T*)b, (T*)o, n)));
    DONE();
}
extern "C" int pk_log_softmax(const void* x, int dtype, long long ld, float* y, long long rows, int n, float scale, void* stream) {
    const int grid = grid_for(rows, 8);
    PK_DISPATCH_T(dtype, (log_softmax_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)x, ld, y, rows, n, scale)));
    DONE();
}
extern "C" int pk_row_lse(const void* x, int dtype, long long ld, float* lse, long long rows, int n, float scale, void* stream) {
    const int grid = grid_for(rows, 8);
    PK_DISPATCH_T(dtype, (log_softmax_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)x, ld, nullptr, rows, n, scale, lse)));
    DONE();
}

template <typename T, int UI>
static void launch_gate_fwd_sliced(const void* ex, const void* py, void* h, int B, int T_, int U1, int H, int ld_h, cudaStream_t st) {
    joint_gate_fwd_sliced_kernel<T, UI><<<B * (H / 32), 128, U1 * 64 * (int)sizeof(T), st>>>((const T*)ex, (const T*)py, (T*)h, B, T_, U1, H, ld_h);
}
extern "C" int pk_joint_gate_fwd(const void* ex, const void* py, void* h, int dtype, int B, int T_, int U1, int H, int ld_h, void* stream) {
    PK_CHECK_ARG(H % 8 == 0 && ld_h % 8 == 0 && ld_h >= H, "H, ld_h must be multiples of 8");
    const int ui = (U1 + 31) / 32;
    if (H % 32 == 0 && ui <= 5 && T_ >= 8) {
        cudaStream_t st = STREAM(stream);
#define PK_GATE_CASE(N) case N: { PK_DISPATCH_T(dtype, (launch_gate_fwd_sliced<T, N>(ex, py, h, B, T_, U1, H, ld_h, st))); } break;
        switch (ui) { PK_GATE_CASE(1) PK_GATE_CASE(2) PK_GATE_CASE(3) PK_GATE_CASE(4) PK_GATE_CASE(5) }
#undef PK_GATE_CASE
        DONE();
    }
    PK_DISPATCH_T(dtype, (joint_gate_fwd_kernel<T><<<B * T_, 128, 0, STREAM(stream)>>>((const T*)ex, (const T*)py, (T*)h, B, T_, U1, H, ld_h)));
    DONE();
}

template <typename T, int UI>
static void launch_gate_bwd_fused(const void* ex, const void* py, const void* dh, const int* dh_map, void* dex, void* dpy, int B, int T_, int U1, int H,
                                  cudaStream_t st) {
    const int smem = U1 * 64 * (int)sizeof(T);
    // (capping the registers for 3 CTAs per SM instead of 2 -- 168 registers, 84 spilled bytes at UI = 5 -- measured slower: 1.77 vs 1.40 ms)
    joint_gate_bwd_fused_kernel<T, UI><<<B * (H / 32), 128, smem, st>>>((const T*)ex, (const T*)py, (const T*)dh, dh_map, (T*)dex, (T*)dpy, B, T_, U1,
                                                                     H);
}
extern "C" int pk_joint_gate_bwd(const void* ex, const void* py, const void* dh, const int* dh_map, void* dex, void* dpy, int dtype, int B,
                                 int T_, int U1, int H, void* stream) {
    PK_CHECK_ARG(H % 8 == 0, "H must be a multiple of 8");
    const int ui = (U1 + 31) / 32;
    if (H % 32 == 0 && ui <= 5) {
        cudaStream_t st = STREAM(stream);
#define PK_GATE_CASE(N) case N: { PK_DISPATCH_T(dtype, (launch_gate_bwd_fused<T, N>(ex, py, dh, dh_map, dex, dpy, B, T_, U1, H, st))); } break;
        switch (ui) { PK_GATE_CASE(1) PK_GATE_CASE(2) PK_GATE_CASE(3) PK_GATE_CASE(4) PK_GATE_CASE(5) }
#undef PK_GATE_CASE
        DONE();
    }
    PK_DISPATCH_T(dtype, (joint_gate_bwd_ex_kernel<T><<<B * T_, 128, 0, STREAM(stream)>>>((const T*)ex, (const T*)py, (const T*)dh, dh_map, (T*)dex, B, T_, U1, H)));
    PK_CHECK_LAUNCH(); count_launch();
    PK_DISPATCH_T(dtype, (joint_gate_bwd_py_kernel<T><<<B * U1, 128, 0, STREAM(stream)>>>((const T*)ex, (const T*)py, (const T*)dh, dh_map, (T*)dpy, B, T_, U1, H)));
    DONE();
}

extern "C" int pk_lstm_cell_fwd(const float* gx, long long ld_gx, const float* gh, long long ld_gh, const float* c_prev, float* c_out,
                                void* h_out, int dtype, long long ld_h, float* gates_save, int B, int H, void* stream) {
    PK_DISPATCH_T(dtype, (lstm_cell_fwd_kernel<T><<<(B * H + 255) / 256, 256, 0, STREAM(stream)>>>(gx, ld_gx, gh, ld_gh, c_prev, c_out,
                                                                                                (T*)h_out, ld_h, gates_save, B, H)));
    DONE();
}
extern "C" int pk_lstm_cell_bwd(const void* dh_out, long long ld_dho, const float* dh_rec, const float* dc_next, const float* gates,
                                const float* c, const float* c_prev, void* dgates, int dtype, float* dc_prev, int B, int H,
                                void* stream) {
    PK_DISPATCH_T(dtype, (lstm_cell_bwd_kernel<T><<<(B * H + 255) / 256, 256, 0, STREAM(stream)>>>((const T*)dh_out, ld_dho, dh_rec, dc_next,
                                                                                                gates, c, c_prev, (T*)dgates, dc_prev, B, H)));
    DONE();
}

extern "C" int pk_embedding_fwd(const long long* idx, const float* table, int E, void* out, int dtype, int ld_out, long long n,
                                void* stream) {
    const int grid = grid_for(n * ld_out, 256);
    PK_DISPATCH_T(dtype, (embedding_fwd_kernel<T><<<grid, 256, 0, STREAM(stream)>>>(idx, table, E, (T*)out, ld_out, n)));
    DONE();
}
extern "C" int pk_embedding_bwd(const long long* idx, const void* dout, int dtype, int ld, int E, float* dtable, long long n,
                                long long padding_idx, void* stream) {
    const int grid = grid_for(n * E, 256);
    PK_DISPATCH_T(dtype, (embedding_bwd_kernel<T><<<grid, 256, 0, STREAM(stream)>>>(idx, (const T*)dout, ld, E, dtable, n, padding_idx)));
    DONE();
}

extern "C" int pk_gather_rows(const void* src, const int* idx, void* dst, int dtype, long long rows, int C, void* stream) {
    PK_CHECK_ARG(C % 8 == 0 && rows > 0, "C must be a multiple of 8 and rows > 0");
    PK_CHECK_ARG(aligned16(src) && aligned16(dst), "pk_gather_rows: src, dst must be 16-byte aligned");
    PK_DISPATCH_T(dtype, (gather_rows_kernel<T><<<(unsigned)rows, 128, 0, STREAM(stream)>>>((const T*)src, idx, (T*)dst, rows, C)));
    DONE();
}
extern "C" int pk_scatter_add_rows(const void* src, const int* idx, float* dst, int dtype, long long rows, int C, void* stream) {
    PK_CHECK_ARG(rows > 0, "rows must be > 0");
    PK_DISPATCH_T(dtype, (scatter_add_rows_kernel<T><<<(unsigned)rows, 256, 0, STREAM(stream)>>>((const T*)src, idx, dst, rows, C)));
    DONE();
}
extern "C" int pk_ce_grad(const void* z, int dtype, long long ld, const int* tok, const float* coef, float scale, void* dz,
                          long long rows, int n, void* stream) {
    PK_CHECK_ARG(rows > 0 && n > 0 && ld >= n, "bad shape");
    const int grid = grid_for(rows, 8);
    PK_DISPATCH_T(dtype, (ce_grad_kernel<T><<<grid, 256, 0, STREAM(stream)>>>((const T*)z, ld, tok, coef, scale, (T*)dz, rows, n)));
    DONE();
}
