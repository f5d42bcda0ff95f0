// Optimiser-side kernels on the flat fp32 parameter vector: inf-norm gradient clipping,
// Nesterov SGD, and the BMUF block-momentum update.  Pure HBM streams (float4, grid-stride).
//
//   trainer/train_transducer_bmuf_otfaug.py:105-110  clip_grad_norm_(inf) + SGD(nesterov).step()
//   trainer/bmuf.py:76-100                            BmufTrainer.update_and_sync
#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ x, long long n, unsigned int* __restrict__ out_bits,
                                                     int* __restrict__ nan_flag) {
    float m = 0.f;
    bool bad = false;
    const long long n4 = n / 4;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = x4[i];
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
        bad |= !(v.x == v.x) | !(v.y == v.y) | !(v.z == v.z) | !(v.w == v.w);
    }
    for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        m = fmaxf(m, fabsf(x[i]));
        bad |= !(x[i] == x[i]);
    }
    m = warp_max(m);
    const bool warp_bad = __any_sync(0xffffffffu, bad);          // all 32 lanes reach this point
    if ((threadIdx.x & 31) == 0) {
        atomicMax(out_bits, __float_as_uint(m));     // non-negative floats order like their bit patterns
        if (nan_flag && warp_bad) atomicExch(nan_flag, 1);
    }
}

// g' = g * min(1, max_norm / (absmax + 1e-6));  buf = first ? g' : mom*buf + g';  p -= lr * (g' + mom*buf)
__global__ void __launch_bounds__(256) sgd_nesterov_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf,
                                                           long long n, float lr, float mom, float max_norm,
                                                           const unsigned int* __restrict__ absmax_bits,
                                                           const int* __restrict__ nan_flag, int first) {
    float coef = 1.f;
    if (max_norm > 0.f && absmax_bits) {
        const float tot = __uint_as_float(*absmax_bits);
        coef = fminf(1.f, max_norm / (tot + 1e-6f));
        // fmaxf drops NaNs, torch.max does not: clip_grad_norm_(inf) of a gradient holding a NaN gives a NaN coefficient,
        // i.e. every parameter turns NaN (and the next BMUF sync stops the run); reproduced through the flag absmax raised
        if (nan_flag && *nan_flag) coef = __int_as_float(0x7fc00000);
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i] * coef;
        const float b = first ? gi : mom * buf[i] + gi;
        buf[i] = b;
        p[i] -= lr * (gi + mom * b);
    }
}

// delta = global - local  (the vector that is sum-reduced across ranks)
__global__ void __launch_bounds__(256) bmuf_delta_kernel(const float* __restrict__ glob, const float* __restrict__ local,
                                                         float* __restrict__ delta, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        delta[i] = glob[i] - local[i];
}
// d = dsum / N; dprev = bm*dprev + blr*(1-bm)*d; glob -= (1+bm)*dprev; local = glob
__global__ void __launch_bounds__(256) bmuf_update_kernel(float* __restrict__ glob, float* __restrict__ local,
                                                          float* __restrict__ dprev, const float* __restrict__ dsum, long long n,
                                                          float inv_world, float bm, float blr) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float d = dsum[i] * inv_world;
        const float dp = bm * dprev[i] + blr * (1.f - bm) * d;
        dprev[i] = dp;
        const float gnew = glob[i] - (1.f + bm) * dp;
        glob[i] = gnew;
        local[i] = gnew;
    }
}

// ---------------------------------------------------------------------------------------------- Adam and BMUF-Adam
// The element formulas spell out torch's roundings with _rn intrinsics, so that nvcc's multiply-add contraction cannot move
// them: fused where torch's CUDA kernels fuse (lerp, addcmul, addcdiv), separate where torch rounds an intermediate tensor.
struct AdamScalars {
    float w1;          // 1 - beta1  (lerp weight)
    float beta2, w2;   // beta2, 1 - beta2
    float bc2_sqrt;    // sqrt(1 - beta2^step)
    float eps;
    float neg_step;    // -lr / (1 - beta1^step)
};

// g' = g * coef;  m.lerp_(g', 1-b1);  v = b2*v + (1-b2)*g'^2;  p += -step_size * m / (sqrt(v)/bc2_sqrt + eps)
// (torch.optim.Adam, foreach path: _foreach_lerp_, _foreach_mul_, _foreach_addcmul_, _foreach_sqrt, _foreach_div_,
// _foreach_add_, _foreach_addcdiv_)
__device__ __forceinline__ float adam_elem(float& p, float g, float& m, float& v, float coef, const AdamScalars& s) {
    const float gc = __fmul_rn(g, coef);
    m = __fmaf_rn(s.w1, __fsub_rn(gc, m), m);                       // lerp with weight < 0.5: self + w * (end - self)
    v = __fmaf_rn(s.w2, __fmul_rn(gc, gc), __fmul_rn(v, s.beta2));  // addcmul: a + value * (b * c)
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), s.bc2_sqrt), s.eps);
    p = __fmaf_rn(s.neg_step, __fdiv_rn(m, den), p);                // addcdiv: a + value * (b / c)
    return p;
}

__device__ __forceinline__ float clip_coef(float max_norm, const unsigned int* absmax_bits, const int* nan_flag) {
    float coef = 1.f;
    if (max_norm > 0.f && absmax_bits) {
        coef = fminf(1.f, max_norm / (__uint_as_float(*absmax_bits) + 1e-6f));
        if (nan_flag && *nan_flag) coef = __int_as_float(0x7fc00000);   // as sgd_nesterov_kernel: torch's NaN coefficient
    }
    return coef;
}

// vec: every pointer 16-byte aligned (the flat buffers' slots are), so the body runs as float4; the n % 4 tail is scalar
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, float* __restrict__ p_out2, long long n, AdamScalars s,
                                                   float max_norm, const unsigned int* __restrict__ absmax_bits,
                                                   const int* __restrict__ nan_flag, int vec) {
    const float coef = clip_coef(max_norm, absmax_bits, nan_flag);
    const long long stride = (long long)gridDim.x * blockDim.x, t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n4 = vec ? n / 4 : 0;
    for (long long i = t; i < n4; i += stride) {
        float4 P = reinterpret_cast<float4*>(p)[i], M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
        const float4 G = reinterpret_cast<const float4*>(g)[i];
        adam_elem(P.x, G.x, M.x, V.x, coef, s);
        adam_elem(P.y, G.y, M.y, V.y, coef, s);
        adam_elem(P.z, G.z, M.z, V.z, coef, s);
        adam_elem(P.w, G.w, M.w, V.w, coef, s);
        reinterpret_cast<float4*>(p)[i] = P;
        reinterpret_cast<float4*>(m)[i] = M;
        reinterpret_cast<float4*>(v)[i] = V;
        if (p_out2) reinterpret_cast<float4*>(p_out2)[i] = P;
    }
    for (long long i = n4 * 4 + t; i < n; i += stride) {
        float pi = p[i], mi = m[i], vi = v[i];
        adam_elem(pi, g[i], mi, vi, coef, s);
        p[i] = pi; m[i] = mi; v[i] = vi;
        if (p_out2) p_out2[i] = pi;
    }
}

// BmufAdamTrainer.update_and_sync's master update (trainer/bmuf.py:274-297, then the broadcast and the copies of :298-321),
// replicated on every rank.  fp32 with the reference's tensor roundings (each scalar * tensor and tensor +- tensor rounded):
//   x = sum / world                                    for delta, m, v
//   dprev = bm * dprev + (blr*(1-bm)) * d;  glob -= (1+bm) * dprev;  local = glob
//   m_g = ((b1t*(b1r-1)) * m_g + (1-b1t*b1r) * m) / (1-b1t);  the same for v_g with beta2;  local moments = m_g, v_g
struct BmufAdamScalars {
    float inv_world, bm, c_blr, one_bm;
    float a1, c1, d1;   // b1t*(b1r-1), 1-b1t*b1r, 1-b1t
    float a2, c2, d2;
};

__device__ __forceinline__ void bmuf_adam_elem(float& glob, float& local, float& dprev, float& mg, float& vg, float dsum, float& m,
                                               float& v, const BmufAdamScalars& s) {
    const float d = __fmul_rn(dsum, s.inv_world), ma = __fmul_rn(m, s.inv_world), va = __fmul_rn(v, s.inv_world);
    dprev = __fadd_rn(__fmul_rn(s.bm, dprev), __fmul_rn(s.c_blr, d));
    glob = __fsub_rn(glob, __fmul_rn(s.one_bm, dprev));
    local = glob;
    mg = __fdiv_rn(__fadd_rn(__fmul_rn(s.a1, mg), __fmul_rn(s.c1, ma)), s.d1);
    vg = __fdiv_rn(__fadd_rn(__fmul_rn(s.a2, vg), __fmul_rn(s.c2, va)), s.d2);
    m = mg;
    v = vg;
}

// msg = [delta_sum; m_sum; v_sum] (3n); its moment slots are overwritten with the new local moments
__global__ void __launch_bounds__(256) bmuf_adam_kernel(float* __restrict__ glob, float* __restrict__ local,
                                                        float* __restrict__ dprev, float* __restrict__ mg, float* __restrict__ vg,
                                                        float* __restrict__ msg, long long n, BmufAdamScalars s, int vec) {
    const long long stride = (long long)gridDim.x * blockDim.x, t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const float* __restrict__ dsum = msg;
    float* __restrict__ m = msg + n;
    float* __restrict__ v = msg + 2 * n;
    const long long n4 = vec ? n / 4 : 0;
    for (long long i = t; i < n4; i += stride) {
        float4 G = reinterpret_cast<float4*>(glob)[i], L, DP = reinterpret_cast<float4*>(dprev)[i];
        float4 MG = reinterpret_cast<float4*>(mg)[i], VG = reinterpret_cast<float4*>(vg)[i];
        float4 M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
        const float4 D = reinterpret_cast<const float4*>(dsum)[i];
        bmuf_adam_elem(G.x, L.x, DP.x, MG.x, VG.x, D.x, M.x, V.x, s);
        bmuf_adam_elem(G.y, L.y, DP.y, MG.y, VG.y, D.y, M.y, V.y, s);
        bmuf_adam_elem(G.z, L.z, DP.z, MG.z, VG.z, D.z, M.z, V.z, s);
        bmuf_adam_elem(G.w, L.w, DP.w, MG.w, VG.w, D.w, M.w, V.w, s);
        reinterpret_cast<float4*>(glob)[i] = G;
        reinterpret_cast<float4*>(local)[i] = L;
        reinterpret_cast<float4*>(dprev)[i] = DP;
        reinterpret_cast<float4*>(mg)[i] = MG;
        reinterpret_cast<float4*>(vg)[i] = VG;
        reinterpret_cast<float4*>(m)[i] = M;
        reinterpret_cast<float4*>(v)[i] = V;
    }
    for (long long i = n4 * 4 + t; i < n; i += stride) {
        float G = glob[i], L, DP = dprev[i], MG = mg[i], VG = vg[i], M = m[i], V = v[i];
        bmuf_adam_elem(G, L, DP, MG, VG, dsum[i], M, V, s);
        glob[i] = G; local[i] = L; dprev[i] = DP; mg[i] = MG; vg[i] = VG; m[i] = M; v[i] = V;
    }
}
}  // namespace pk

using namespace pk;
static int og(long long n) {
    long long g = (n + 1023) / 1024, cap = (long long)num_sms() * 8;
    return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

/* out_bits[0] must be zeroed by the caller (cudaMemsetAsync) -- done here. nan_flag (int*, may be NULL) is set to 1 on NaN. */
extern "C" int pk_absmax(const float* x, long long n, float* out, int* nan_flag, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    PK_CHECK_CUDA(cudaMemsetAsync(out, 0, 4, st));
    absmax_kernel<<<og(n), 256, 0, st>>>(x, n, reinterpret_cast<unsigned int*>(out), nan_flag);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_sgd_nesterov_clip(float* p, const float* g, float* buf, long long n, float lr, float momentum, float max_norm,
                                    const float* absmax, const int* nan_flag, int first, void* stream) {
    sgd_nesterov_kernel<<<og(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, g, buf, n, lr, momentum, max_norm,
                                                                                 reinterpret_cast<const unsigned int*>(absmax), nan_flag, first);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_bmuf_delta(const float* glob, const float* local, float* delta, long long n, void* stream) {
    bmuf_delta_kernel<<<og(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(glob, local, delta, n);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
extern "C" int pk_bmuf_update(float* glob, float* local, float* delta_prev, const float* delta_sum, long long n, int world,
                              float block_momentum, float block_lr, void* stream) {
    PK_CHECK_ARG(world >= 1, "world must be >= 1");
    bmuf_update_kernel<<<og(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(glob, local, delta_prev, delta_sum, n, 1.f / world,
                                                                                block_momentum, block_lr);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int pk_adam_clip(float* p, const float* g, float* exp_avg, float* exp_avg_sq, float* p_out2, long long n, double lr,
                            double beta1, double beta2, double eps, double bias_correction1, double bias_correction2_sqrt,
                            float max_norm, const float* absmax, const int* nan_flag, void* stream) {
    PK_CHECK_ARG(n >= 0, "n must be >= 0");
    PK_CHECK_ARG(bias_correction1 > 0.0 && bias_correction2_sqrt > 0.0, "bias corrections must be > 0 (step > 0)");
    if (n == 0) return 0;
    AdamScalars s;
    s.w1 = (float)(1.0 - beta1);
    s.beta2 = (float)beta2;
    s.w2 = (float)(1.0 - beta2);
    s.bc2_sqrt = (float)bias_correction2_sqrt;
    s.eps = (float)eps;
    s.neg_step = (float)((lr / bias_correction1) * -1.0);
    const int vec = aligned16(p) && aligned16(g) && aligned16(exp_avg) && aligned16(exp_avg_sq) && (!p_out2 || aligned16(p_out2));
    adam_kernel<<<og(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, g, exp_avg, exp_avg_sq, p_out2, n, s, max_norm,
                                                                          reinterpret_cast<const unsigned int*>(absmax), nan_flag, vec);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_bmuf_adam_update(float* glob, float* local, float* delta_prev, float* exp_avg_g, float* exp_avg_sq_g, float* msg,
                                   long long n, int world, double block_momentum, double block_lr, double beta1_tau,
                                   double beta1_rho, double beta2_tau, double beta2_rho, void* stream) {
    PK_CHECK_ARG(world >= 1, "world must be >= 1");
    PK_CHECK_ARG(n >= 0, "n must be >= 0");
    PK_CHECK_ARG(beta1_tau < 1.0 && beta2_tau < 1.0, "beta^sync_period must be < 1");
    if (n == 0) return 0;
    BmufAdamScalars s;
    s.inv_world = 1.f / (float)world;
    s.bm = (float)block_momentum;
    s.c_blr = (float)(block_lr * (1.0 - block_momentum));
    s.one_bm = (float)(1.0 + block_momentum);
    s.a1 = (float)(beta1_tau * (beta1_rho - 1.0));
    s.c1 = (float)(1.0 - beta1_tau * beta1_rho);
    s.d1 = (float)(1.0 - beta1_tau);
    s.a2 = (float)(beta2_tau * (beta2_rho - 1.0));
    s.c2 = (float)(1.0 - beta2_tau * beta2_rho);
    s.d2 = (float)(1.0 - beta2_tau);
    // the moment slots msg + n, msg + 2n are float4-aligned when msg is and n % 4 == 0
    const int vec = aligned16(glob) && aligned16(local) && aligned16(delta_prev) && aligned16(exp_avg_g) && aligned16(exp_avg_sq_g) &&
                    aligned16(msg) && n % 4 == 0;
    bmuf_adam_kernel<<<og(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(glob, local, delta_prev, exp_avg_g, exp_avg_sq_g, msg,
                                                                                n, s, vec);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}
