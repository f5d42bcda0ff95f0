// Shared device helpers for the pika_b200 sm_90a kernels: PTX wrappers for mbarrier, TMA
// (cp.async.bulk.tensor), wgmma, plus small numeric utilities.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define PK_DEVICE __device__ __forceinline__

namespace pk {

// ---------------------------------------------------------------- error plumbing (host)
void set_last_error(const char* fmt, ...);
#define PK_CHECK_ARG(cond, msg)                                       \
    do {                                                              \
        if (!(cond)) {                                                \
            pk::set_last_error("%s:%d: %s", __FILE__, __LINE__, msg); \
            return -1;                                                \
        }                                                             \
    } while (0)
#define PK_CHECK_CUDA(expr)                                                                     \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            pk::set_last_error("%s:%d: CUDA error %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return -2;                                                                          \
        }                                                                                       \
    } while (0)
#define PK_CHECK_LAUNCH() PK_CHECK_CUDA(cudaGetLastError())

int num_sms();
int encode_tiled_bf16_3d(CUtensorMap* out, const void* ptr, const unsigned long long (&dims)[3], const unsigned long long (&strides_bytes)[2],
                         const unsigned (&box)[3], const char* what);

// ---------------------------------------------------------------- dtype helpers
enum DType : int { F32 = 0, BF16 = 1 };

template <typename T> PK_DEVICE float to_f32(T v);
template <> PK_DEVICE float to_f32<float>(float v) { return v; }
template <> PK_DEVICE float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> PK_DEVICE T from_f32(float v);
template <> PK_DEVICE float from_f32<float>(float v) { return v; }
template <> PK_DEVICE __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

PK_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
PK_DEVICE float ex2_approx(float x) {            // 2^x on the MUFU, flush-to-zero, no range fix-up (2^-inf = 0)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
PK_DEVICE float bf16lo(uint32_t v) { return __uint_as_float(v << 16); }
PK_DEVICE float bf16hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

// activation pair of the gated joint (dense and pruned): precise libm in the fp32-class mode, MUFU.TANH in production (bf16)
template <typename T> PK_DEVICE float jt_tanh(float x);
template <> PK_DEVICE float jt_tanh<float>(float x) { return tanhf(x); }
template <> PK_DEVICE float jt_tanh<__nv_bfloat16>(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
template <typename T> PK_DEVICE float jt_sigmoid(float x);
template <> PK_DEVICE float jt_sigmoid<float>(float x) { return 1.f / (1.f + expf(-x)); }
template <> PK_DEVICE float jt_sigmoid<__nv_bfloat16>(float x) { return fmaf(jt_tanh<__nv_bfloat16>(0.5f * x), 0.5f, 0.5f); }

// Counter-based dropout RNG: a 64-bit element index and a seed -> 32 uniform bits.
// (murmur3-style finaliser; forward and backward regenerate the same mask.)
PK_DEVICE uint32_t hash_u32(uint64_t idx, uint32_t seed) {
    uint32_t x = (uint32_t)idx ^ (seed * 0x9E3779B9u);
    uint32_t y = (uint32_t)(idx >> 32) + seed;
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    x += y * 0x85ebca6bU;
    x ^= x >> 13; x *= 0xc2b2ae35U; x ^= x >> 16;
    return x;
}
// keep iff hash >= thresh where thresh = p * 2^32
PK_DEVICE bool drop_keep(uint64_t idx, uint32_t seed, uint32_t thresh) { return hash_u32(idx, seed) >= thresh; }

// Attention-probability dropout: one hash per PAIR of adjacent keys of a probability row, 16 bits per element.  The mask is the
// largest integer-ALU item of the fused attention kernels, so the per-pair part is kept to seven instructions: a per-row salt
// (full-strength hash of the row index, computed once per row) plus a two-round multiply / xor-shift of (salt + pair index).
// `salt` = drop_row_salt(row of the [B*heads*T, T] probability matrix, seed); kp = key >> 1; returns keep bits (bit 0: even key,
// bit 1: odd key).  keep iff the 16-bit lane >= thresh16 = round(p * 65536); the keep-scale is 1 / (1 - thresh16 / 65536).
PK_DEVICE uint32_t drop_row_salt(uint64_t grow, uint32_t seed) { return hash_u32(grow, seed); }
PK_DEVICE uint32_t drop_pair(uint32_t salt, uint32_t kp, uint32_t thresh16) {
    uint32_t x = (salt + kp) * 0x9E3779B1u;
    x ^= x >> 15; x *= 0x85EBCA77u; x ^= x >> 13;
    return ((x & 0xFFFFu) >= thresh16 ? 1u : 0u) | ((x >> 16) >= thresh16 ? 2u : 0u);
}
__host__ __device__ inline uint32_t drop_thresh16_of(float p) {
    if (p <= 0.f) return 0u;
    const double t = (double)p * 65536.0 + 0.5;
    const uint32_t r = t >= 65535.0 ? 65535u : (uint32_t)t;
    return r == 0 ? 1u : r;
}
__host__ __device__ inline float drop_scale16_of(uint32_t thresh16) { return thresh16 ? 1.f / (1.f - (float)thresh16 / 65536.f) : 1.f; }

// Chunk mask of streaming self-attention (DESIGN.md "Chunked attention"): frame t lies in chunk (t + off) / len, and query i sees key j
// iff chunk(i) - left <= chunk(j) <= chunk(i) (left = -1: no lower limit).  Allowed keys [lo, hi) of query i and allowed queries
// [lo, hi) of key j, clipped to [0, T); each end is monotone in i (j).
__host__ __device__ inline int chunk_clip(long long v, int T) { return (int)(v < 0 ? 0 : v > T ? T : v); }
__host__ __device__ inline int chunk_key_lo(int i, int T, int len, int off, int left) {
    return left < 0 ? 0 : chunk_clip(((long long)((i + (long long)off) / len) - left) * len - off, T);
}
__host__ __device__ inline int chunk_key_hi(int i, int T, int len, int off) { return chunk_clip(((i + (long long)off) / len + 1) * len - off, T); }
__host__ __device__ inline int chunk_query_lo(int j, int T, int len, int off) { return chunk_clip((j + (long long)off) / len * len - off, T); }
__host__ __device__ inline int chunk_query_hi(int j, int T, int len, int off, int left) {
    return left < 0 ? T : chunk_clip(((j + (long long)off) / len + left + 1) * len - off, T);
}

PK_DEVICE float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
PK_DEVICE float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- PTX: shared address, election
PK_DEVICE uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

PK_DEVICE bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b32 r;\n\t"
        "elect.sync r|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- PTX: mbarrier
PK_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
PK_DEVICE void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
PK_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
PK_DEVICE void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
PK_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
PK_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---------------------------------------------------------------- PTX: TMA
PK_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
PK_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
PK_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// plain (non-tensor) bulk copy global -> shared, bytes % 16 == 0, both addresses 16-byte aligned
PK_DEVICE void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
PK_DEVICE void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
            reinterpret_cast<uint64_t>(m)),
        "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
PK_DEVICE void tma_reduce_add_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
            reinterpret_cast<uint64_t>(m)),
        "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// L2 eviction-priority policies (the encodings createpolicy.fractional.L2::evict_{normal,first,last} produce for fraction 1.0)
constexpr uint64_t kL2EvictNormal = 0x1000000000000000ull;
constexpr uint64_t kL2EvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kL2EvictLast = 0x14F0000000000000ull;
PK_DEVICE void tma_load_4d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol)
        : "memory");
}
PK_DEVICE void tma_store_4d_hint(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group.L2::cache_hint [%0, {%2, %3, %4, %5}], [%1], %6;" ::"l"(
            reinterpret_cast<uint64_t>(m)),
        "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol)
        : "memory");
}
PK_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> PK_DEVICE void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N> PK_DEVICE void tma_store_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
PK_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- PTX: wgmma (warpgroup MMA, sm_90a)
// Shared-memory matrix descriptor (sm_90), SWIZZLE_128B:
//   bits [0,14)  start address >> 4          bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4     bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major tiles (rows of 64 bf16 = 128 B, 8-row atoms of 1024 B): LBO unused (1), SBO = 1024, a k16 step adds 32 B.
// MN-major tiles (64-wide MN chunks of k-rows): LBO = distance between MN chunks, SBO = 1024 (8 k-rows), a k16 step adds 2048 B.
PK_DEVICE uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
PK_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
PK_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> PK_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R> PK_DEVICE void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N> PK_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> PK_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// D (+)= A * B on one warpgroup, m64 x N x k16, bf16 inputs, fp32 accumulators in registers (acc = 0: D = A * B).
// TA / TB: 1 = the operand is MN-major in shared memory.  Accumulator register i of thread t holds
//   row (t / 32) * 16 + (t % 32) / 4 + 8 * ((i >> 1) & 1), column (i >> 2) * 8 + (t % 4) * 2 + (i & 1).
// The _rs form takes A from registers: four bf16 pairs laid out like the accumulator of an m64 x 16 product.
template <int TA, int TB> PK_DEVICE void wgmma_ss_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <int TB> PK_DEVICE void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc), "n"(TB));
}
template <int TA, int TB> PK_DEVICE void wgmma_ss_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB> PK_DEVICE void wgmma_ss_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

// ---------------------------------------------------------------- PTX: thread-block clusters
PK_DEVICE uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
PK_DEVICE uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
PK_DEVICE void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------- predicated single-lane issue
// The producer warps run their loops CONVERGED (all 32 lanes wait on the barriers and compute the same addresses) and only the
// asynchronous instruction itself is predicated on one elected lane.  Inside an `if (lane == 0)` region the compiler has to wrap every
// instruction that takes uniform-register operands (UTMALDG) in an elect / R2UR / BRA.U.ANY loop.
PK_DEVICE uint32_t elect_one_u32() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b32 r;\n\t"
        "elect.sync r|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(pred));
    return pred;
}
PK_DEVICE void mbar_arrive_expect_tx_p(uint64_t* bar, uint32_t bytes, uint32_t pred) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}\n" ::"r"(smem_u32(bar)),
                 "r"(bytes), "r"(pred)
                 : "memory");
}
PK_DEVICE void tma_load_3d_p(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %6, 0;\n\t"
        "@q cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}\n" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(pred)
        : "memory");
}
PK_DEVICE void bulk_load_p(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %4, 0;\n\t"
        "@q cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}\n" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar)), "r"(pred)
        : "memory");
}
PK_DEVICE void tma_load_4d_hint_p(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3, uint64_t pol, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %8, 0;\n\t"
        "@q cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;\n\t}\n" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol), "r"(pred)
        : "memory");
}
PK_DEVICE void tma_store_4d_hint_p(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3, uint64_t pol, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %7, 0;\n\t"
        "@q cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group.L2::cache_hint [%0, {%2, %3, %4, %5}], [%1], %6;\n\t}\n" ::"l"(
            reinterpret_cast<uint64_t>(m)),
        "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol), "r"(pred)
        : "memory");
}
PK_DEVICE void tma_reduce_add_4d_p(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %6, 0;\n\t"
        "@q cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n\t}\n" ::"l"(
            reinterpret_cast<uint64_t>(m)),
        "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(pred)
        : "memory");
}
PK_DEVICE void tma_store_commit_p(uint32_t pred) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %0, 0;\n\t@q cp.async.bulk.commit_group;\n\t}\n" ::"r"(pred) : "memory");
}
template <int N> PK_DEVICE void tma_store_wait_read_p(uint32_t pred) {
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %1, 0;\n\t@q cp.async.bulk.wait_group.read %0;\n\t}\n" ::"n"(N), "r"(pred) : "memory");
}

PK_DEVICE void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---------------------------------------------------------------- PTX: shared-memory loads / stores
// stores four 8 x 8 bf16 matrices; register i holds the thread's two elements of matrix i in the mma fragment layout (row lane / 4,
// columns 2 * (lane % 4) + {0, 1}); lanes 8i .. 8i + 7 give the 16-byte row addresses of matrix i
PK_DEVICE void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}
PK_DEVICE uint4 lds_u32x4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
PK_DEVICE uint2 lds_u32x2(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
    return v;
}
PK_DEVICE float2 lds_f32x2(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}
PK_DEVICE void sts_f32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
PK_DEVICE uint32_t bf16x2_max(uint32_t a, uint32_t b) {      // lane-wise max of two bf16 pairs (a NaN loses to a number)
    uint32_t d;
    asm("max.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}

}  // namespace pk
