// On-the-fly front end on the GPU: speed perturbation + RMS gain + int16 quantisation, Kaldi-compatible
// fbank, splice + padding + CMN/CMVN + SpecAugment.  One batch = a handful of launches.
//
//   loader/audio.py:28-36,207-262,551-603      AudioSegment.{change_speed, normalize, gain_db, rms_db, _convert_*}
//   loader/otf_utt_loader.py:195-201,218-234   augmentation chain + PyKaldi Fbank.compute_features (egs/fbank.conf)
//   loader/otf_utt_loader.py:28-46,262-270     splice +-ctx with edge replication; pad with the last valid frame
//   trainer/train_transducer_bmuf_otfaug.py:86-93 + utils/spec_augment.py:10-20   CMN (padded axis), CMVN, SpecAugment
//
// Integer path (augmented int16 samples): the speed-perturbed branch follows numpy's float64 arithmetic
// (no FMA contraction) and is bit-exact up to the summation order of the mean square (1e-16 relative);
// the rate == 1.0 branch stays in float32 like numpy, where the mean square is accumulated in float64
// here versus numpy's float32 pairwise sum, so individual samples may differ by 1 LSB (see DESIGN.md).
#include <math.h>

#include "../../include/pika_b200.h"
#include "common.cuh"

namespace pk {
void count_launch();

constexpr int AUG_THREADS = 256;

// ------------------------------------------------------------------------------------ augmentation
// pass A: resample (float64, numpy.interp semantics) and per-CTA partial sums of squares
__global__ void __launch_bounds__(AUG_THREADS) aug_resample_kernel(const short* __restrict__ pcm, long long ld_pcm,
                                                                   const int* __restrict__ n_samples, const float* __restrict__ rate,
                                                                   const int* __restrict__ new_len, double* __restrict__ resampled,
                                                                   long long ld_res, double* __restrict__ partial, int parts) {
    const int b = blockIdx.y;
    const int N = n_samples[b], L = new_len[b];
    const short* src = pcm + (long long)b * ld_pcm;
    double* dst = resampled + (long long)b * ld_res;
    const bool unit = (rate[b] == 1.0f);
    const double step = (L > 1) ? (double)N / (double)(L - 1) : 0.0;      // numpy.linspace(0, N, L)
    double acc = 0.0;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x) {
        double v;
        if (unit) {
            const float s = (float)src[j] * (1.0f / 32768.0f);
            v = (double)s;
            const float sq = s * s;                                      // numpy: float32 array ** 2
            acc += (double)sq;
        } else {
            const double x = (j == L - 1 && L > 1) ? (double)N : __dmul_rn((double)j, step);   // linspace(0, N, 1) = [0]
            if (x >= (double)(N - 1)) {
                v = (double)((float)src[N - 1] * (1.0f / 32768.0f));     // right of the last knot: fp[-1]
            } else {
                const int i = (int)x;                                    // floor, x >= 0
                const double f0 = (double)((float)src[i] * (1.0f / 32768.0f));
                const double f1 = (double)((float)src[i + 1] * (1.0f / 32768.0f));
                const double slope = __dsub_rn(f1, f0);                  // (f1-f0)/(1.0)
                v = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, (double)i)), f0);
            }
            acc += __dmul_rn(v, v);
        }
        dst[j] = v;
    }
    // deterministic block reduction (fixed tree), one partial per CTA
    __shared__ double red[AUG_THREADS];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = AUG_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[(long long)b * parts + blockIdx.x] = red[0];
}

// AudioSegment.normalize(target_db) gain from the per-CTA partial sums of squares (fixed summation order)
PK_DEVICE double normalize_gain(const double* __restrict__ partial, int parts, int L, bool unit, double target_db, int* err_flag) {
    double tot = 0.0;
    for (int i = 0; i < parts; ++i) tot += partial[i];
    double ms = (L > 0) ? tot / (double)L : 0.0;
    if (unit) ms = (double)(float)ms;                                    // numpy float32 mean
    ms = fmax(1e-20, ms);
    const double rms_db = 10.0 * log10(ms);
    double gain_db = target_db - rms_db;
    if (gain_db > 300.0) { atomicExch(err_flag, 1); gain_db = 300.0; }  // reference raises ValueError
    return pow(10.0, gain_db / 20.0);
}

// _convert_samples_from_float32(.., 'int16'): scale by 2^15, clip, C-cast truncation toward zero
PK_DEVICE int quantise(double s, double gain, bool unit) {
    if (unit) {
        float v = __fmul_rn((float)s, (float)gain);
        v = __fmul_rn(v, 32768.0f);
        v = fminf(fmaxf(v, -32768.0f), 32767.0f);
        return (int)v;
    }
    double v = __dmul_rn(s, gain);
    v = __dmul_rn(v, 32768.0);
    v = fmin(fmax(v, -32768.0), 32767.0);
    return (int)v;
}

// pass B: gain from the mean square, apply, quantise to int16 (stored as float for the fbank kernel)
__global__ void __launch_bounds__(AUG_THREADS) aug_gain_kernel(const double* __restrict__ resampled, long long ld_res,
                                                               const double* __restrict__ partial, int parts,
                                                               const float* __restrict__ rate, const int* __restrict__ new_len,
                                                               const float* __restrict__ target_db, float* __restrict__ wave,
                                                               short* __restrict__ wave_i16, long long ld_wave, int* __restrict__ err_flag) {
    const int b = blockIdx.y;
    const int L = new_len[b];
    const bool unit = (rate[b] == 1.0f);
    __shared__ double s_gain;
    if (threadIdx.x == 0) s_gain = normalize_gain(partial + (long long)b * parts, parts, L, unit, (double)target_db[b], err_flag);
    __syncthreads();
    const double gain = s_gain;
    const double* src = resampled + (long long)b * ld_res;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x) {
        const int q = quantise(src[j], gain, unit);
        wave[(long long)b * ld_wave + j] = (float)q;
        if (wave_i16) wave_i16[(long long)b * ld_wave + j] = (short)q;
    }
}

// ------------------------------------------------------------------------------------ noise + reverberation
//   loader/audio.py:426-513  AudioSegment.{add_noise, convolve_and_normalize}; call sites loader/otf_utt_loader.py:224-228
// On these paths the gained signal stays in the float64 workspace (float32-valued on the rate == 1.0 branch, where the
// reference's samples are float32) until the final renormalise + quantise pass.

// fixed-tree CTA reduction; thread 0 writes the CTA's partial
template <int THREADS>
PK_DEVICE void cta_partial(double acc, double* __restrict__ out) {
    __shared__ double red[THREADS];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = red[0];
}

// rms_db of a signal from its partial sums of squares; float32 arithmetic on the rate == 1.0 branch like numpy's
PK_DEVICE double rms_db_of(const double* __restrict__ partial, int parts, int L, bool unit) {
    double tot = 0.0;
    for (int i = 0; i < parts; ++i) tot += partial[i];
    double ms = (L > 0) ? tot / (double)L : 0.0;
    if (unit) ms = (double)(float)ms;
    ms = fmax(1e-20, ms);
    const double db = 10.0 * log10(ms);
    return unit ? (double)(float)db : db;
}

// pass B': the gain of pass B, applied in place and kept in float; partial sums of squares of the gained signal
__global__ void __launch_bounds__(AUG_THREADS) aug_gain_keep_kernel(double* __restrict__ sig, long long ld_sig,
                                                                    const double* __restrict__ partial, int parts,
                                                                    const float* __restrict__ rate, const int* __restrict__ new_len,
                                                                    const float* __restrict__ target_db, double* __restrict__ partial_out,
                                                                    int* __restrict__ err_flag) {
    const int b = blockIdx.y;
    const int L = new_len[b];
    const bool unit = (rate[b] == 1.0f);
    __shared__ double s_gain;
    if (threadIdx.x == 0) s_gain = normalize_gain(partial + (long long)b * parts, parts, L, unit, (double)target_db[b], err_flag);
    __syncthreads();
    const double gain = s_gain;
    double* x = sig + (long long)b * ld_sig;
    double acc = 0.0;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x) {
        if (unit) {
            const float v = __fmul_rn((float)x[j], (float)gain);
            x[j] = (double)v;
            acc += (double)__fmul_rn(v, v);
        } else {
            const double v = __dmul_rn(x[j], gain);
            x[j] = v;
            acc += __dmul_rn(v, v);
        }
    }
    cta_partial<AUG_THREADS>(acc, partial_out + (long long)b * gridDim.x + blockIdx.x);
}

// add_noise: noise gain min(rms_db - noise_rms_db - snr, 300) dB on the float32 noise slice (float64 multiply, float32
// result, as numpy's in-place float32 *= float64), superimposed; partial sums of squares of the noisy signal
__global__ void __launch_bounds__(AUG_THREADS) aug_noise_kernel(double* __restrict__ sig, long long ld_sig, const double* __restrict__ partial,
                                                                int parts, const float* __restrict__ rate, const int* __restrict__ new_len,
                                                                const short* __restrict__ noise, const int* __restrict__ noise_idx,
                                                                const long long* __restrict__ noise_off, const double* __restrict__ snr,
                                                                const double* __restrict__ noise_rms_db, double* __restrict__ partial_out) {
    const int b = blockIdx.y;
    const int L = new_len[b];
    const bool unit = (rate[b] == 1.0f);
    __shared__ double s_gain;
    if (threadIdx.x == 0) {
        const double sig_db = rms_db_of(partial + (long long)b * parts, parts, L, unit);
        const double nz_db = noise_rms_db[noise_idx[b]];
        const double diff = unit ? (double)__fsub_rn((float)sig_db, (float)nz_db) : sig_db - nz_db;
        s_gain = pow(10.0, fmin(diff - snr[b], 300.0) / 20.0);
    }
    __syncthreads();
    const double gain = s_gain;
    double* x = sig + (long long)b * ld_sig;
    const short* nz = noise + noise_off[b];
    double acc = 0.0;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x) {
        const float n = (float)__dmul_rn((double)((float)nz[j] * (1.0f / 32768.0f)), gain);
        if (unit) {
            const float v = __fadd_rn((float)x[j], n);
            x[j] = (double)v;
            acc += (double)__fmul_rn(v, v);
        } else {
            const double v = __dadd_rn(x[j], (double)n);
            x[j] = v;
            acc += __dmul_rn(v, v);
        }
    }
    cta_partial<AUG_THREADS>(acc, partial_out + (long long)b * gridDim.x + blockIdx.x);
}

// renormalise to the pre-convolution rms_db (convolve_and_normalize) when post != nullptr, then quantise as pass B
__global__ void __launch_bounds__(AUG_THREADS) aug_renorm_quant_kernel(const double* __restrict__ sig, long long ld_sig,
                                                                       const double* __restrict__ pre, int pre_parts,
                                                                       const double* __restrict__ post, int post_parts,
                                                                       const float* __restrict__ rate, const int* __restrict__ new_len,
                                                                       float* __restrict__ wave, short* __restrict__ wave_i16,
                                                                       long long ld_wave, int* __restrict__ err_flag) {
    const int b = blockIdx.y;
    const int L = new_len[b];
    const bool unit = (rate[b] == 1.0f);
    __shared__ double s_gain;
    if (threadIdx.x == 0) {
        double gain = 1.0;
        if (post) {
            const double t_db = rms_db_of(pre + (long long)b * pre_parts, pre_parts, L, unit);
            const double c_db = rms_db_of(post + (long long)b * post_parts, post_parts, L, unit);
            double gain_db = unit ? (double)__fsub_rn((float)t_db, (float)c_db) : t_db - c_db;
            if (gain_db > 300.0) { atomicExch(err_flag, 1); gain_db = 300.0; }
            gain = pow(10.0, gain_db / 20.0);
        }
        s_gain = gain;
    }
    __syncthreads();
    const double gain = s_gain;
    const double* src = sig + (long long)b * ld_sig;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x) {
        const int q = quantise(src[j], gain, unit);
        wave[(long long)b * ld_wave + j] = (float)q;
        if (wave_i16) wave_i16[(long long)b * ld_wave + j] = (short)q;
    }
}

// ---- fftconvolve(x, h, "same") in float64: uniformly partitioned overlap-save, FFT size 2*Lb.
// y[n] = sum_m h[m] x[n + c - m], c = (M-1)//2, n in [0, N).  With x'[i] = x[i + c] and h_p = h[p*Lb, (p+1)*Lb):
// output block j (Lb samples) = last Lb samples of IFFT(sum_p H_p . X_{j-p}), X_q = FFT of x'[(q-1)*Lb, (q+1)*Lb).
// Real inputs: only bins 0..Lb of each spectrum are stored; the inverse restores the rest by Hermitian symmetry.
constexpr int CONV_THREADS = 512;

struct RirF64 {             // ragged float64 RIRs, one per signal
    const double* h; long long ld; const int* len;
    PK_DEVICE int length(int b) const { return len[b]; }
    PK_DEVICE double at(int b, int i) const { return h[(long long)b * ld + i]; }
};
struct RirBank {            // int16 bank; signal b uses RIR idx[b] (float32 samples, x 2^-15)
    const short* bank; const long long* off; const int* len; const int* idx;
    PK_DEVICE int length(int b) const { return len[idx[b]]; }
    PK_DEVICE double at(int b, int i) const { return (double)((float)bank[off[idx[b]] + i] * (1.0f / 32768.0f)); }
};

struct ConvGeom {
    int lb, log2n, p_max, j_max, q_max;     // q index = q + p_max - 1, in [0, q_max)
};

PK_DEVICE double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// in-place radix-2 DIT on bit-reversed input in shared memory; tw[k] = exp(-2 pi i k / n), k < n/2
template <bool INV>
PK_DEVICE void fft_smem(double2* buf, int log2n, const double2* __restrict__ tw) {
    const int half_n = 1 << (log2n - 1);
    for (int s = 1; s <= log2n; ++s) {
        const int half = 1 << (s - 1);
        for (int t = threadIdx.x; t < half_n; t += blockDim.x) {
            const int pos = t & (half - 1);
            const int i0 = ((t >> (s - 1)) << s) + pos, i1 = i0 + half;
            double2 w = tw[pos << (log2n - s)];
            if (INV) w.y = -w.y;
            const double2 a = buf[i0], c = cmul(buf[i1], w);
            buf[i0] = make_double2(a.x + c.x, a.y + c.y);
            buf[i1] = make_double2(a.x - c.x, a.y - c.y);
        }
        __syncthreads();
    }
}

PK_DEVICE int brev(int i, int log2n) { return (int)(__brev((unsigned)i) >> (32 - log2n)); }

__global__ void conv_twiddle_kernel(double2* __restrict__ tw, int n) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n / 2) {
        double s, c;
        sincospi(2.0 * (double)k / (double)n, &s, &c);
        tw[k] = make_double2(c, -s);
    }
}

// H[b][p] for p < ceil(M_b / Lb)
template <typename Rir>
__global__ void __launch_bounds__(CONV_THREADS) conv_rir_spectra_kernel(Rir rir, ConvGeom g, const double2* __restrict__ tw,
                                                                        double2* __restrict__ H) {
    extern __shared__ double2 cbuf[];
    const int p = blockIdx.x, b = blockIdx.y, n = 2 * g.lb;
    const int M = rir.length(b);
    if (p * g.lb >= M) return;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int m = p * g.lb + i;
        cbuf[brev(i, g.log2n)] = make_double2((i < g.lb && m < M) ? rir.at(b, m) : 0.0, 0.0);
    }
    __syncthreads();
    fft_smem<false>(cbuf, g.log2n, tw);
    double2* dst = H + ((long long)b * g.p_max + p) * (g.lb + 1);
    for (int k = threadIdx.x; k <= g.lb; k += blockDim.x) dst[k] = cbuf[k];
}

// X[b][q] for the blocks that some output block reads: -(P_b - 1) <= q < J_b
template <typename Rir>
__global__ void __launch_bounds__(CONV_THREADS) conv_signal_spectra_kernel(const double* __restrict__ x, long long ld_x,
                                                                           const int* __restrict__ n_len, Rir rir, ConvGeom g,
                                                                           const double2* __restrict__ tw, double2* __restrict__ X) {
    extern __shared__ double2 cbuf[];
    const int qi = blockIdx.x, b = blockIdx.y, n = 2 * g.lb;
    const int q = qi - (g.p_max - 1);
    const int N = n_len[b], M = rir.length(b);
    const int J = (N + g.lb - 1) / g.lb, P = (M + g.lb - 1) / g.lb;
    if (q >= J || q < -(P - 1)) return;
    const long long base = (long long)(q - 1) * g.lb + (M - 1) / 2;
    const double* xs = x + (long long)b * ld_x;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const long long s = base + i;
        cbuf[brev(i, g.log2n)] = make_double2((s >= 0 && s < N) ? xs[s] : 0.0, 0.0);
    }
    __syncthreads();
    fft_smem<false>(cbuf, g.log2n, tw);
    double2* dst = X + ((long long)b * g.q_max + qi) * (g.lb + 1);
    for (int k = threadIdx.x; k <= g.lb; k += blockDim.x) dst[k] = cbuf[k];
}

// output block j: accumulate over partitions per bin, inverse FFT, keep the last Lb samples.  `unit` (nullable): signals with
// rate == 1.0 are rounded to float32, as the reference's float32 fftconvolve returns.  Optional partial sums of squares
// per block (0 for blocks past the signal's end).
template <typename Rir>
__global__ void __launch_bounds__(CONV_THREADS) conv_accum_inverse_kernel(const double2* __restrict__ H, const double2* __restrict__ X,
                                                                          const int* __restrict__ n_len, Rir rir, ConvGeom g,
                                                                          const double2* __restrict__ tw, const float* __restrict__ rate,
                                                                          double* __restrict__ y, long long ld_y,
                                                                          double* __restrict__ partial) {
    extern __shared__ double2 cbuf[];
    const int j = blockIdx.x, b = blockIdx.y, n = 2 * g.lb;
    const int N = n_len[b], M = rir.length(b);
    const int J = (N + g.lb - 1) / g.lb, P = min((M + g.lb - 1) / g.lb, g.p_max);
    if (j >= J) {
        if (partial && threadIdx.x == 0) partial[(long long)b * g.j_max + j] = 0.0;
        return;
    }
    const double2* Hb = H + (long long)b * g.p_max * (g.lb + 1);
    const double2* Xb = X + (long long)b * g.q_max * (g.lb + 1);
    for (int k = threadIdx.x; k <= g.lb; k += blockDim.x) {
        double2 acc = make_double2(0.0, 0.0);
#pragma unroll 2
        for (int p = 0; p < P; ++p) {
            const double2 h = Hb[(long long)p * (g.lb + 1) + k];
            const double2 xv = Xb[(long long)(j - p + g.p_max - 1) * (g.lb + 1) + k];
            acc.x = fma(h.x, xv.x, fma(-h.y, xv.y, acc.x));
            acc.y = fma(h.x, xv.y, fma(h.y, xv.x, acc.y));
        }
        cbuf[brev(k, g.log2n)] = acc;
        if (k > 0 && k < g.lb) cbuf[brev(n - k, g.log2n)] = make_double2(acc.x, -acc.y);
    }
    __syncthreads();
    fft_smem<true>(cbuf, g.log2n, tw);
    const bool unit = rate && rate[b] == 1.0f;
    const double inv_n = 1.0 / (double)n;
    double* ys = y + (long long)b * ld_y;
    double acc = 0.0;
    for (int i = threadIdx.x; i < g.lb; i += blockDim.x) {
        const int o = j * g.lb + i;
        if (o >= N) break;
        double v = cbuf[g.lb + i].x * inv_n;
        if (unit) {
            const float f = (float)v;
            v = (double)f;
            acc += (double)__fmul_rn(f, f);
        } else {
            acc += v * v;
        }
        ys[o] = v;
    }
    if (partial) cta_partial<CONV_THREADS>(acc, partial + (long long)b * g.j_max + j);
}

// ------------------------------------------------------------------------------------ fbank
// FFT sizes 2^7 .. 2^11: 8 to 48 kHz at frames up to 42 ms (--round-to-power-of-two)
constexpr int FB_LOG2_MIN = 7, FB_LOG2_MAX = 11;

struct FbankTables {
    const float* window;    // [frame_len] window function
    const float2* twiddle;  // [N/2] exp(-2 pi i k / N)
    const float* mel_w;     // [n_mel][N/2]
    const int* mel_lo;      // [n_mel] first non-zero bin
    const int* mel_hi;      // [n_mel] one past the last non-zero bin
};

struct FrameGeom {          // Kaldi FrameExtractionOptions, in samples
    int frame_len, frame_shift, snip_edges, remove_dc;
};

struct MfccParams {         // Kaldi MfccOptions past the mel banks (feat/feature-mfcc.cc); unused by the fbank instances
    const float* dct;       // [n_mel][num_ceps]: DCT-II rows times the lifter, transposed so that a frame's coefficients read coalesced
    int num_ceps, use_energy, raw_energy, htk_compat;
    float energy_floor;     // floor of the energy when > 0 (linear, as --energy-floor)
};

// N/2 butterflies per stage, one per thread; at least 256 threads so that every mel bin (n_mel <= 256) has one
constexpr int fbank_threads(int log2n) { return (1 << (log2n - 1)) < 256 ? 256 : (1 << (log2n - 1)); }

// standard normal from two counter-based hashes (Box-Muller); one draw per (utterance, frame, sample), as Kaldi's Dither() draws
// one RandGauss() per sample of every extracted window (feat/feature-window.cc: Dither) -- its RNG stream itself is not reproducible
PK_DEVICE float dither_gauss(uint64_t idx, uint32_t seed) {
    const uint32_t h1 = hash_u32(idx * 2, seed), h2 = hash_u32(idx * 2 + 1, seed ^ 0x6A09E667u);
    const float u1 = ((float)h1 + 1.0f) * 2.3283064365386963e-10f;          // (0, 1]
    const float u2 = (float)h2 * 2.3283064365386963e-10f;
    return sqrtf(-2.f * __logf(u1)) * __cosf(6.283185307179586f * u2);
}

// Kaldi's ExtractWindow at snip_edges = false: samples outside [0, n) are reflected about the signal's edges until inside
PK_DEVICE long long reflect_index(long long s, long long n) {
    while (s < 0 || s >= n) s = s < 0 ? -s - 1 : 2 * n - 1 - s;
    return s;
}

// one CTA per (frame, utterance), a full SM's worth of threads resident.  n_len: samples per utterance (read only when
// snip_edges = 0).  THREADS >= N/2, so every loop below has a trip count known at compile time.  The arithmetic is spelled out with
// explicit roundings: DC removal fused into the subtraction of the window's sum times -1/frame_len, pre-emphasis as
// fma(-c, prev, cur), the complex products and |X|^2 with the first product fused -- the same operations, in the same order, at
// every FFT size.
//
// MFCC = true swaps the epilogue for Kaldi's MfccComputer::Compute: the log mel energies go to shared memory and each of the first
// num_ceps threads forms one cepstral coefficient, then the frame's log energy replaces c0 (use_energy) and HTK ordering moves c0 last.
// The energy is summed per thread in the pre-emphasis loop, after dither and DC removal (raw_energy, Kaldi's ProcessWindow) or of the
// windowed frame (otherwise).  The fbank instances (MFCC = false) compile to the code they had before the epilogue was added.
template <int LOG2N, bool MFCC>
__global__ void __launch_bounds__(fbank_threads(LOG2N), 2048 / fbank_threads(LOG2N)) fbank_kernel(const float* __restrict__ wave, long long ld_wave,
                                                                     const int* __restrict__ n_len, const int* __restrict__ n_frames,
                                                                     FbankTables tb, FrameGeom g, int n_mel, float preemph,
                                                                     float* __restrict__ feats, long long ld_b, int t_max, float dither,
                                                                     uint32_t dither_seed, MfccParams mp) {
    constexpr int N = 1 << LOG2N, NB = N / 2, THREADS = fbank_threads(LOG2N), WARPS = THREADS / 32;
    constexpr int PER_THREAD = (N + THREADS - 1) / THREADS;
    const int t = blockIdx.x, b = blockIdx.y;
    if (t >= n_frames[b]) return;
    __shared__ float2 buf[N];
    __shared__ float frame[N];
    __shared__ float red[WARPS];
    __shared__ float power[NB];
    const int tid = threadIdx.x, L = g.frame_len;
    const float* src = wave + (long long)b * ld_wave;
    const uint64_t key = ((uint64_t)b * (uint64_t)t_max + (uint64_t)t) * (uint64_t)L;
    float part = 0.f;
    if (g.snip_edges) {
        src += (long long)t * g.frame_shift;
#pragma unroll
        for (int j = 0; j < PER_THREAD; ++j) {
            const int i = tid + j * THREADS;
            if (i < L) {
                float v = src[i];
                if (dither != 0.f) v = __fmaf_rn(dither, dither_gauss(key + (uint64_t)i, dither_seed), v);
                frame[i] = v; part += v;
            }
        }
    } else {
        const long long start = (long long)t * g.frame_shift + g.frame_shift / 2 - L / 2, n = n_len[b];
#pragma unroll
        for (int j = 0; j < PER_THREAD; ++j) {
            const int i = tid + j * THREADS;
            if (i < L) {
                float v = src[reflect_index(start + i, n)];
                if (dither != 0.f) v = __fmaf_rn(dither, dither_gauss(key + (uint64_t)i, dither_seed), v);
                frame[i] = v; part += v;
            }
        }
    }
    part = warp_sum(part);
    if ((tid & 31) == 0) red[tid >> 5] = part;
    __syncthreads();
    float sum = 0.f, neg_inv_len = 0.f;
    if (g.remove_dc) {
#pragma unroll
        for (int w = 0; w < WARPS; ++w) sum += red[w];
        neg_inv_len = -(1.0f / (float)L);
    }
    // DC removal, pre-emphasis (x[i] -= c*x[i-1], x[0] -= c*x[0]), window, zero-pad, bit-reversed placement
    float energy = 0.f;                                 // MFCC: this thread's part of the frame's sum of squares
#pragma unroll
    for (int j = 0; j < PER_THREAD; ++j) {
        const int i = tid + j * THREADS;
        if (i < N) {
            float v = 0.f;
            if (i < L) {
                const float cur = __fmaf_rn(sum, neg_inv_len, frame[i]);
                const float prev = __fmaf_rn(sum, neg_inv_len, i > 0 ? frame[i - 1] : frame[0]);
                v = __fmul_rn(__fmaf_rn(-preemph, prev, cur), tb.window[i]);
                if constexpr (MFCC) {
                    const float x = mp.raw_energy ? cur : v;
                    energy = __fmaf_rn(x, x, energy);
                }
            }
            const int r = __brev((unsigned)i) >> (32 - LOG2N);
            buf[r] = make_float2(v, 0.f);
        }
    }
    __shared__ float ered[MFCC ? WARPS : 1];
    if constexpr (MFCC) {
        energy = warp_sum(energy);
        if ((tid & 31) == 0) ered[tid >> 5] = energy;   // read after the FFT's barriers
    }
    __syncthreads();
    // LOG2N radix-2 stages of N/2 butterflies, one per thread
#pragma unroll
    for (int s = 1; s <= LOG2N; ++s) {
        if (NB == THREADS || tid < NB) {
            const int half = 1 << (s - 1);
            const int grp = tid >> (s - 1), pos = tid & (half - 1);
            const int i0 = grp * (half << 1) + pos, i1 = i0 + half;
            const float2 w = tb.twiddle[pos << (LOG2N - s)];
            const float2 a = buf[i0], c = buf[i1];
            const float2 wc = make_float2(__fmaf_rn(c.x, w.x, -__fmul_rn(c.y, w.y)), __fmaf_rn(c.x, w.y, __fmul_rn(c.y, w.x)));
            buf[i0] = make_float2(__fadd_rn(a.x, wc.x), __fadd_rn(a.y, wc.y));
            buf[i1] = make_float2(__fsub_rn(a.x, wc.x), __fsub_rn(a.y, wc.y));
        }
        __syncthreads();
    }
    if (NB == THREADS || tid < NB) power[tid] = __fmaf_rn(buf[tid].x, buf[tid].x, __fmul_rn(buf[tid].y, buf[tid].y));
    __syncthreads();
    __shared__ float logmel[MFCC ? 256 : 1];
    if (tid < n_mel) {
        float e = 0.f;
        const float* w = tb.mel_w + (long long)tid * NB;
        for (int k = tb.mel_lo[tid]; k < tb.mel_hi[tid]; ++k) e = __fmaf_rn(w[k], power[k], e);
        if constexpr (MFCC)
            logmel[tid] = logf(fmaxf(e, 1.1920928955078125e-07f));
        else
            feats[(long long)b * ld_b + (long long)t * n_mel + tid] = logf(fmaxf(e, 1.1920928955078125e-07f));
    }
    if constexpr (MFCC) {
        __syncthreads();
        const int nc = mp.num_ceps;
        if (tid < nc) {
            float c = 0.f;
            for (int j = 0; j < n_mel; ++j) c = __fmaf_rn(mp.dct[j * nc + tid], logmel[j], c);
            if (tid == 0) {
                if (mp.use_energy) {
                    float e = 0.f;
#pragma unroll
                    for (int w = 0; w < WARPS; ++w) e += ered[w];
                    c = logf(fmaxf(e, 1.1920928955078125e-07f));
                    if (mp.energy_floor > 0.f) c = fmaxf(c, logf(mp.energy_floor));
                } else if (mp.htk_compat) {
                    c = __fmul_rn(c, 1.41421356237309505f);
                }
            }
            const int col = mp.htk_compat ? (tid == 0 ? nc - 1 : tid - 1) : tid;
            feats[(long long)b * ld_b + (long long)t * nc + col] = c;
        }
    }
}

// ------------------------------------------------------------------------------------ splice / CMN / CMVN / SpecAugment
// output row t of the padded batch: splice(feats)[::stride] (n_out = ceil(n_frames / stride) rows), rows >= n_out replicating the
// last one; the spliced row of fbank frame tt stacks frames tt-lctx .. tt+rctx, clamped to the utterance.  STRIDED = false is
// stride 1 without the extra index arithmetic, which costs the splice kernels about 13 % (they are instruction-bound)
template <bool STRIDED>
PK_DEVICE float spliced_value(const float* __restrict__ fb, int n_frames, int n_out, int n_mel, int lctx, int stride, int t, int col) {
    const int tt = STRIDED ? min(t, n_out - 1) * stride : min(t, n_frames - 1);
    const int k = col / n_mel, c = col - k * n_mel;
    int src = tt + k - lctx;
    src = max(0, min(n_frames - 1, src));
    return fb[(long long)src * n_mel + c];
}
// CMN column sums in a fixed order, so that the mean does not depend on the order in which CTAs finish: each CTA sums its 64 rows
// in row order into partial [B, parts, D] (parts = gridDim.x), then splice_colmerge adds the parts in block order
template <bool STRIDED>
__global__ void splice_colsum_kernel(const float* __restrict__ feats, long long ld_b, const int* __restrict__ n_frames, int n_mel,
                                     int lctx, int stride, int D, int t_max, float* __restrict__ partial) {
    const int b = blockIdx.y, col = threadIdx.x;
    if (col >= D || n_frames[b] <= 0) return;
    const int t0 = blockIdx.x * 64, t1 = min(t_max, t0 + 64);
    const float* fb = feats + (long long)b * ld_b;
    const int nf = n_frames[b], n_out = STRIDED ? (nf + stride - 1) / stride : nf;
    float s = 0.f;
    for (int t = t0; t < t1; ++t) s += spliced_value<STRIDED>(fb, nf, n_out, n_mel, lctx, stride, t, col);
    partial[((long long)b * gridDim.x + blockIdx.x) * D + col] = s;
}
// sums [B, D] <- the parts of splice_colsum added in block order (0 for an utterance without frames, whose parts are not written)
__global__ void splice_colmerge_kernel(const float* __restrict__ partial, int parts, const int* __restrict__ n_frames, int D,
                                       float* __restrict__ sums) {
    const int b = blockIdx.x, col = threadIdx.x;
    if (col >= D) return;
    float s = 0.f;
    if (n_frames[b] > 0)
        for (int p = 0; p < parts; ++p) s += partial[((long long)b * parts + p) * D + col];
    sums[(long long)b * D + col] = s;
}
template <typename T, bool STRIDED>
__global__ void splice_finalize_kernel(const float* __restrict__ feats, long long ld_b, const int* __restrict__ n_frames, int n_mel,
                                       int lctx, int stride, int D, int t_max, const float* __restrict__ sums, int cmn,
                                       const float* __restrict__ offset, const float* __restrict__ scale, int f0, int fs, int t0m,
                                       int ts, T* __restrict__ out) {
    const int b = blockIdx.y;
    const long long total = (long long)t_max * D;
    const float* fb = feats + (long long)b * ld_b;
    const int nf = n_frames[b], n_out = STRIDED ? (nf + stride - 1) / stride : nf;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i / D), col = (int)(i - (long long)t * D);
        float v = nf > 0 ? spliced_value<STRIDED>(fb, nf, n_out, n_mel, lctx, stride, t, col) : 0.f;
        if (cmn) v -= sums[(long long)b * D + col] / (float)t_max;
        if (offset) { v += offset[col]; v *= scale[col]; }
        if ((fs > 0 && col >= f0 && col < f0 + fs) || (ts > 0 && t >= t0m && t < t0m + ts)) v = 0.f;
        out[(long long)b * total + i] = from_f32<T>(v);
    }
}
}  // namespace pk

using namespace pk;

/* Workspace layout of pk_frontend_fwd: resampled f64 [B, n_max] | partial f64 [B, parts] | wave f32 [B, n_max] |
 * feats f32 [B, t_max, n_mel] | sums f32 [B, D] | CMN partials f32 [B, ceil(t_max / 64), D] | err int.  t_max here counts fbank
 * frames, before the splice's stride, so it bounds the output rows the CMN sums run over. */
static const int kAugParts = 64;
static long long cmn_parts(long long t_max) { return (t_max + 63) / 64; }
extern "C" long long pk_frontend_workspace_bytes(int B, int n_max, int t_max, int n_mel, int D) {
    long long b = 0;
    b += (long long)B * n_max * 8 + (long long)B * kAugParts * 8;
    b += (long long)B * n_max * 4;
    b += (long long)B * t_max * n_mel * 4;
    b += (long long)B * D * 4 + (long long)B * cmn_parts(t_max) * D * 4 + 256;
    return b + 1024;
}

/* ---- float64 same-mode convolution (overlap-save), shared by pk_conv_same_f64 and the front end's reverberation stage.
 * Workspace: twiddles [Lb] | H [B, P_max, Lb+1] | X [B, J_max + P_max - 1, Lb+1], complex f64, each 256-byte aligned. */
static const int kRirMaxLen = 65536;
static long long align256(long long b) { return (b + 255) & ~255LL; }

// block length: a power of two in [1024, 4096], about a quarter of the longest RIR (HBM traffic of the accumulation ~ 16 N M / Lb)
static int conv_block_len(int m_max) {
    int lb = 1024;
    while (lb < 4096 && 4 * lb < m_max) lb <<= 1;
    return lb;
}
static ConvGeom conv_geom(int n_max, int m_max) {
    ConvGeom g;
    g.lb = conv_block_len(m_max);
    g.log2n = 1;
    while ((1 << g.log2n) < 2 * g.lb) ++g.log2n;
    g.p_max = (m_max + g.lb - 1) / g.lb;
    g.j_max = (n_max + g.lb - 1) / g.lb;
    g.q_max = g.j_max + g.p_max - 1;
    return g;
}
static long long conv_ws_bytes(int B, const ConvGeom& g) {
    return align256((long long)g.lb * 16) + align256((long long)B * g.p_max * (g.lb + 1) * 16) +
           align256((long long)B * g.q_max * (g.lb + 1) * 16);
}

// y [B, ld_y] <- same-mode convolution of x (lengths n_len) with rir; y may alias x.  Partial sums of squares per Lb block into
// partial [B, J_max] when non-null.
template <typename Rir>
static int conv_same_launch(const double* x, long long ld_x, const int* n_len, Rir rir, int B, const ConvGeom& g, const float* rate,
                            double* y, long long ld_y, double* partial, unsigned char* ws, cudaStream_t st) {
    double2* tw = reinterpret_cast<double2*>(ws);
    ws += align256((long long)g.lb * 16);
    double2* H = reinterpret_cast<double2*>(ws);
    ws += align256((long long)B * g.p_max * (g.lb + 1) * 16);
    double2* X = reinterpret_cast<double2*>(ws);
    const int smem = 2 * g.lb * (int)sizeof(double2);
    PK_CHECK_CUDA(cudaFuncSetAttribute(conv_rir_spectra_kernel<Rir>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    PK_CHECK_CUDA(cudaFuncSetAttribute(conv_signal_spectra_kernel<Rir>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    PK_CHECK_CUDA(cudaFuncSetAttribute(conv_accum_inverse_kernel<Rir>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    conv_twiddle_kernel<<<(g.lb + 255) / 256, 256, 0, st>>>(tw, 2 * g.lb);
    PK_CHECK_LAUNCH(); count_launch();
    conv_rir_spectra_kernel<Rir><<<dim3(g.p_max, B), CONV_THREADS, smem, st>>>(rir, g, tw, H);
    PK_CHECK_LAUNCH(); count_launch();
    conv_signal_spectra_kernel<Rir><<<dim3(g.q_max, B), CONV_THREADS, smem, st>>>(x, ld_x, n_len, rir, g, tw, X);
    PK_CHECK_LAUNCH(); count_launch();
    conv_accum_inverse_kernel<Rir><<<dim3(g.j_max, B), CONV_THREADS, smem, st>>>(H, X, n_len, rir, g, tw, rate, y, ld_y, partial);
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" long long pk_conv_same_f64_workspace_bytes(int B, int n_max, int m_max) {
    if (B <= 0 || n_max <= 0 || m_max < 1 || m_max > kRirMaxLen) return -1;
    return conv_ws_bytes(B, conv_geom(n_max, m_max));
}

extern "C" int pk_conv_same_f64(const double* x, long long ld_x, const int* n_len, const double* h, long long ld_h, const int* m_len,
                                int B, int n_max, int m_max, double* y, long long ld_y, void* workspace, long long workspace_bytes,
                                void* stream) {
    PK_CHECK_ARG(B > 0 && n_max > 0 && m_max >= 1 && m_max <= kRirMaxLen, "bad conv dims (1 <= m_max <= 65536)");
    const ConvGeom g = conv_geom(n_max, m_max);
    PK_CHECK_ARG(workspace_bytes >= conv_ws_bytes(B, g), "conv workspace too small");
    return conv_same_launch(x, ld_x, n_len, RirF64{h, ld_h, m_len}, B, g, nullptr, y, ld_y, nullptr,
                            reinterpret_cast<unsigned char*>(workspace), reinterpret_cast<cudaStream_t>(stream));
}

/* Noise / RIR banks of pk_frontend_fwd_noise_rir (either may be absent: noise == nullptr / rir == nullptr). */
struct NoiseRirArgs {
    const short* noise; const int* noise_idx; const long long* noise_off; const double* snr; const double* noise_rms_db;
    const short* rir; const long long* rir_off; const int* rir_len; const int* rir_idx; int rir_max_len;
};

/* Workspace of the noise / reverberation path: that of pk_frontend_fwd | partial f64 [B, parts] x 2 | conv partial f64 [B, J_max] |
 * convolution workspace */
static long long noise_rir_extra_bytes(int B, int n_max, int rir_max_len, ConvGeom* g_out) {
    const ConvGeom g = conv_geom(n_max, rir_max_len);
    if (g_out) *g_out = g;
    return 2 * align256((long long)B * kAugParts * 8) + align256((long long)B * g.j_max * 8) + conv_ws_bytes(B, g);
}

extern "C" long long pk_frontend_noise_rir_workspace_bytes(int B, int n_max, int t_max, int n_mel, int D, int rir_max_len) {
    if (rir_max_len < 1 || rir_max_len > kRirMaxLen) return -1;
    return align256(pk_frontend_workspace_bytes(B, n_max, t_max, n_mel, D)) + noise_rir_extra_bytes(B, n_max, rir_max_len, nullptr);
}

// Kaldi fbank frame geometry: FFT size 2^log2_nfft in [2^7, 2^11], 1 <= frame_len <= N, frame_shift >= 1
static bool fbank_geom_ok(int frame_len, int frame_shift, int log2_nfft) {
    return log2_nfft >= FB_LOG2_MIN && log2_nfft <= FB_LOG2_MAX && frame_len >= 1 && frame_len <= (1 << log2_nfft) && frame_shift >= 1;
}

// mp == nullptr: fbank, feats [B, t_max, n_mel]; otherwise MFCC, feats [B, t_max, num_ceps]
template <int LOG2N>
static void fbank_launch_n(const float* wave, long long ld_wave, const int* n_len, const int* n_frames, int B, int t_max,
                           const FbankTables& tb, const FrameGeom& g, int n_mel, float preemph, float* feats, float dither,
                           uint32_t dither_seed, const MfccParams* mp, cudaStream_t st) {
    const dim3 grid(t_max, B);
    if (!mp)
        fbank_kernel<LOG2N, false><<<grid, fbank_threads(LOG2N), 0, st>>>(wave, ld_wave, n_len, n_frames, tb, g, n_mel, preemph, feats,
                                                                          (long long)t_max * n_mel, t_max, dither, dither_seed,
                                                                          MfccParams{});
    else
        fbank_kernel<LOG2N, true><<<grid, fbank_threads(LOG2N), 0, st>>>(wave, ld_wave, n_len, n_frames, tb, g, n_mel, preemph, feats,
                                                                         (long long)t_max * mp->num_ceps, t_max, dither, dither_seed, *mp);
}

// feats <- fbank (mp == nullptr) or MFCC of wave; the geometry has been checked by fbank_geom_ok, the MFCC arguments by mfcc_ok
static int fbank_launch(const float* wave, long long ld_wave, const int* n_len, const int* n_frames, int B, int t_max, const float* window,
                        const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi, int frame_len, int frame_shift,
                        int log2_nfft, int snip_edges, int remove_dc, int n_mel, float preemph, float* feats, float dither,
                        uint32_t dither_seed, cudaStream_t st, const MfccParams* mp = nullptr) {
    const FbankTables tb{window, reinterpret_cast<const float2*>(twiddle), mel_w, mel_lo, mel_hi};
    const FrameGeom g{frame_len, frame_shift, snip_edges ? 1 : 0, remove_dc ? 1 : 0};
    switch (log2_nfft) {
        case 7: fbank_launch_n<7>(wave, ld_wave, n_len, n_frames, B, t_max, tb, g, n_mel, preemph, feats, dither, dither_seed, mp, st); break;
        case 8: fbank_launch_n<8>(wave, ld_wave, n_len, n_frames, B, t_max, tb, g, n_mel, preemph, feats, dither, dither_seed, mp, st); break;
        case 9: fbank_launch_n<9>(wave, ld_wave, n_len, n_frames, B, t_max, tb, g, n_mel, preemph, feats, dither, dither_seed, mp, st); break;
        case 10: fbank_launch_n<10>(wave, ld_wave, n_len, n_frames, B, t_max, tb, g, n_mel, preemph, feats, dither, dither_seed, mp, st); break;
        case 11: fbank_launch_n<11>(wave, ld_wave, n_len, n_frames, B, t_max, tb, g, n_mel, preemph, feats, dither, dither_seed, mp, st); break;
        default: PK_CHECK_ARG(false, "FFT size outside [128, 2048]");
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

// the MFCC epilogue's arguments: 1 <= num_ceps <= n_mel (Kaldi: "num-ceps cannot be larger than num-mel-bins"), a DCT table
static bool mfcc_ok(const MfccParams& mp, int n_mel) {
    return mp.dct && mp.num_ceps >= 1 && mp.num_ceps <= n_mel;
}

// the launch sequence of every front-end entry point; nr == nullptr is pk_frontend_fwd (gain and quantisation in one pass), mp == nullptr
// fbank features (n_mel per frame), otherwise MFCC (num_ceps per frame).  t_max is the number of output rows; the fbank runs over
// t_max * stride frames, which bounds every n_frames[b].
static int frontend_launch(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                           const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx, int rctx,
                           int stride, const float* window, const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi,
                           int frame_len, int frame_shift, int log2_nfft, int snip_edges, int remove_dc, float preemph, int cmn,
                           const float* offset, const float* scale, int f0, int fs, int t0, int ts, void* out, int out_dtype,
                           short* wave_i16_out, void* workspace, long long workspace_bytes, int* err_flag, float dither,
                           unsigned int dither_seed, void* stream, const NoiseRirArgs* nr, const MfccParams* mp = nullptr) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    PK_CHECK_ARG(!mp || mfcc_ok(*mp, n_mel), "bad MFCC arguments (1 <= num_ceps <= n_mel and a DCT table)");
    const int n_feat = mp ? mp->num_ceps : n_mel;     // per-frame width of the features the splice reads
    const int D = n_feat * (lctx + 1 + rctx);
    PK_CHECK_ARG(B > 0 && n_max > 0 && t_max > 0 && n_mel > 0 && n_mel <= 256 && D <= 1024, "bad frontend dims");
    PK_CHECK_ARG(fbank_geom_ok(frame_len, frame_shift, log2_nfft), "bad fbank geometry (FFT size 128..2048, 1 <= frame_len <= FFT size)");
    PK_CHECK_ARG(!snip_edges || n_max >= frame_len, "n_max shorter than one frame");
    PK_CHECK_ARG(stride >= 1 && (long long)t_max * stride <= 0x7fffffffLL, "bad splice stride");
    const int t_fb = t_max * stride;
    PK_CHECK_ARG(workspace_bytes >= pk_frontend_workspace_bytes(B, n_max, t_fb, n_feat, D), "frontend workspace too small");
    ConvGeom g{};
    if (nr) {
        PK_CHECK_ARG(nr->rir_max_len >= 1 && nr->rir_max_len <= kRirMaxLen, "rir_max_len must be in [1, 65536]");
        PK_CHECK_ARG(workspace_bytes >= align256(pk_frontend_workspace_bytes(B, n_max, t_fb, n_feat, D)) +
                                            noise_rir_extra_bytes(B, n_max, nr->rir_max_len, &g),
                     "frontend workspace too small");
    }
    unsigned char* w = reinterpret_cast<unsigned char*>(workspace);
    double* resampled = reinterpret_cast<double*>(w); w += (long long)B * n_max * 8;
    double* partial = reinterpret_cast<double*>(w);   w += (long long)B * kAugParts * 8;
    float* wave = reinterpret_cast<float*>(w);        w += (long long)B * n_max * 4;
    float* feats = reinterpret_cast<float*>(w);       w += (long long)B * t_fb * n_feat * 4;
    float* sums = reinterpret_cast<float*>(w);        w += (long long)B * D * 4;
    float* cmn_part = reinterpret_cast<float*>(w);
    dim3 ga(kAugParts, B);
    aug_resample_kernel<<<ga, AUG_THREADS, 0, st>>>(pcm, ld_pcm, n_samples, rate, new_len, resampled, n_max, partial, kAugParts);
    PK_CHECK_LAUNCH(); count_launch();
    if (!nr) {
        aug_gain_kernel<<<ga, AUG_THREADS, 0, st>>>(resampled, n_max, partial, kAugParts, rate, new_len, target_db, wave, wave_i16_out,
                                                   n_max, err_flag);
        PK_CHECK_LAUNCH(); count_launch();
    } else {
        const long long base = align256(pk_frontend_workspace_bytes(B, n_max, t_fb, n_feat, D));    // checked above, with g
        unsigned char* x = reinterpret_cast<unsigned char*>(workspace) + base;
        double* part_gain = reinterpret_cast<double*>(x);  x += align256((long long)B * kAugParts * 8);
        double* part_noisy = reinterpret_cast<double*>(x); x += align256((long long)B * kAugParts * 8);
        double* part_conv = reinterpret_cast<double*>(x);  x += align256((long long)B * g.j_max * 8);
        aug_gain_keep_kernel<<<ga, AUG_THREADS, 0, st>>>(resampled, n_max, partial, kAugParts, rate, new_len, target_db, part_gain, err_flag);
        PK_CHECK_LAUNCH(); count_launch();
        const double* pre = part_gain;
        if (nr->noise) {
            aug_noise_kernel<<<ga, AUG_THREADS, 0, st>>>(resampled, n_max, part_gain, kAugParts, rate, new_len, nr->noise, nr->noise_idx,
                                                        nr->noise_off, nr->snr, nr->noise_rms_db, part_noisy);
            PK_CHECK_LAUNCH(); count_launch();
            pre = part_noisy;
        }
        if (nr->rir) {
            RirBank bank{nr->rir, nr->rir_off, nr->rir_len, nr->rir_idx};
            if (conv_same_launch(resampled, n_max, new_len, bank, B, g, rate, resampled, n_max, part_conv, x, st)) return 1;
        }
        aug_renorm_quant_kernel<<<ga, AUG_THREADS, 0, st>>>(resampled, n_max, pre, kAugParts, nr->rir ? part_conv : nullptr, g.j_max, rate,
                                                           new_len, wave, wave_i16_out, n_max, err_flag);
        PK_CHECK_LAUNCH(); count_launch();
    }
    if (fbank_launch(wave, n_max, new_len, n_frames, B, t_fb, window, twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift, log2_nfft,
                     snip_edges, remove_dc, n_mel, preemph, feats, dither, dither_seed, st, mp))
        return -1;
    const long long ld_fb = (long long)t_fb * n_feat;
    if (cmn) {
        const int parts = (int)cmn_parts(t_max);
        const dim3 grid(parts, B);
        const int threads = ((D + 31) / 32) * 32;
        if (stride == 1)
            splice_colsum_kernel<false><<<grid, threads, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, cmn_part);
        else
            splice_colsum_kernel<true><<<grid, threads, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, cmn_part);
        PK_CHECK_LAUNCH(); count_launch();
        splice_colmerge_kernel<<<B, threads, 0, st>>>(cmn_part, parts, n_frames, D, sums);
        PK_CHECK_LAUNCH(); count_launch();
    }
    const dim3 grid((int)(((long long)t_max * D + 255) / 256), B);
    if (out_dtype == PK_BF16) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
        if (stride == 1)
            splice_finalize_kernel<__nv_bfloat16, false><<<grid, 256, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, sums,
                                                                               cmn, offset, scale, f0, fs, t0, ts, o);
        else
            splice_finalize_kernel<__nv_bfloat16, true><<<grid, 256, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, sums,
                                                                              cmn, offset, scale, f0, fs, t0, ts, o);
    } else {
        float* o = reinterpret_cast<float*>(out);
        if (stride == 1)
            splice_finalize_kernel<float, false><<<grid, 256, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, sums, cmn,
                                                                       offset, scale, f0, fs, t0, ts, o);
        else
            splice_finalize_kernel<float, true><<<grid, 256, 0, st>>>(feats, ld_fb, n_frames, n_feat, lctx, stride, D, t_max, sums, cmn,
                                                                      offset, scale, f0, fs, t0, ts, o);
    }
    PK_CHECK_LAUNCH(); count_launch();
    return 0;
}

extern "C" int pk_frontend_fwd(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                               const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                               int rctx, int stride, const float* window, const float* twiddle, const float* mel_w, const int* mel_lo,
                               const int* mel_hi, int frame_len, int frame_shift, int log2_nfft, int snip_edges, int remove_dc,
                               float preemph, int cmn, const float* offset, const float* scale, int f0, int fs, int t0, int ts, void* out,
                               int out_dtype, short* wave_i16_out, void* workspace, long long workspace_bytes, int* err_flag,
                               float dither, unsigned int dither_seed, void* stream) {
    return frontend_launch(pcm, ld_pcm, n_samples, rate, new_len, target_db, n_frames, B, n_max, t_max, n_mel, lctx, rctx, stride, window,
                           twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift, log2_nfft, snip_edges, remove_dc, preemph, cmn, offset,
                           scale, f0, fs, t0, ts, out, out_dtype, wave_i16_out, workspace, workspace_bytes, err_flag, dither, dither_seed,
                           stream, nullptr);
}

extern "C" int pk_frontend_fwd_noise_rir(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                                         const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                                         int rctx, int stride, const float* window, const float* twiddle, const float* mel_w,
                                         const int* mel_lo, const int* mel_hi, int frame_len, int frame_shift, int log2_nfft,
                                         int snip_edges, int remove_dc, float preemph, int cmn, const float* offset, const float* scale,
                                         int f0, int fs, int t0, int ts, void* out, int out_dtype, short* wave_i16_out, void* workspace,
                                         long long workspace_bytes, int* err_flag, float dither, unsigned int dither_seed, void* stream,
                                         const short* noise, const int* noise_idx, const long long* noise_off, const double* snr,
                                         const double* noise_rms_db, const short* rir, const long long* rir_off, const int* rir_len,
                                         const int* rir_idx, int rir_max_len) {
    PK_CHECK_ARG(!noise || (noise_idx && noise_off && snr && noise_rms_db), "noise bank without its per-utterance draws");
    PK_CHECK_ARG(!rir || (rir_off && rir_len && rir_idx), "RIR bank without its offsets, lengths or per-utterance draws");
    const NoiseRirArgs nr{noise, noise_idx, noise_off, snr, noise_rms_db, rir, rir_off, rir_len, rir_idx, rir_max_len};
    return frontend_launch(pcm, ld_pcm, n_samples, rate, new_len, target_db, n_frames, B, n_max, t_max, n_mel, lctx, rctx, stride, window,
                           twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift, log2_nfft, snip_edges, remove_dc, preemph, cmn, offset,
                           scale, f0, fs, t0, ts, out, out_dtype, wave_i16_out, workspace, workspace_bytes, err_flag, dither, dither_seed,
                           stream, &nr);
}

/* feats-only entry (fbank of already-augmented int16-scaled samples), used by parity tests and by
 * utils/compute_global_cmvn-style tooling: wave f32 [B, ld_wave] -> feats f32 [B, t_max, n_mel]. */
extern "C" int pk_fbank(const float* wave, long long ld_wave, const int* n_samples, const int* n_frames, int B, int t_max, int n_mel,
                        const float* window, const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi, int frame_len,
                        int frame_shift, int log2_nfft, int snip_edges, int remove_dc, float preemph, float* feats, float dither,
                        unsigned int dither_seed, void* stream) {
    PK_CHECK_ARG(B > 0 && t_max > 0 && n_mel > 0 && n_mel <= 256, "bad fbank dims");
    PK_CHECK_ARG(fbank_geom_ok(frame_len, frame_shift, log2_nfft), "bad fbank geometry (FFT size 128..2048, 1 <= frame_len <= FFT size)");
    PK_CHECK_ARG(snip_edges || n_samples, "snip_edges = 0 needs the sample counts");
    return fbank_launch(wave, ld_wave, n_samples, n_frames, B, t_max, window, twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift,
                        log2_nfft, snip_edges, remove_dc, n_mel, preemph, feats, dither, dither_seed,
                        reinterpret_cast<cudaStream_t>(stream));
}

/* MFCC counterpart of pk_fbank: wave f32 [B, ld_wave] -> feats f32 [B, t_max, num_ceps] */
extern "C" int pk_mfcc(const float* wave, long long ld_wave, const int* n_samples, const int* n_frames, int B, int t_max, int n_mel,
                       const float* window, const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi, int frame_len,
                       int frame_shift, int log2_nfft, int snip_edges, int remove_dc, float preemph, float* feats, float dither,
                       unsigned int dither_seed, void* stream, const float* dct, int num_ceps, int use_energy, int raw_energy,
                       float energy_floor, int htk_compat) {
    const MfccParams mp{dct, num_ceps, use_energy ? 1 : 0, raw_energy ? 1 : 0, htk_compat ? 1 : 0, energy_floor};
    PK_CHECK_ARG(B > 0 && t_max > 0 && n_mel > 0 && n_mel <= 256, "bad fbank dims");
    PK_CHECK_ARG(mfcc_ok(mp, n_mel), "bad MFCC arguments (1 <= num_ceps <= n_mel and a DCT table)");
    PK_CHECK_ARG(fbank_geom_ok(frame_len, frame_shift, log2_nfft), "bad fbank geometry (FFT size 128..2048, 1 <= frame_len <= FFT size)");
    PK_CHECK_ARG(snip_edges || n_samples, "snip_edges = 0 needs the sample counts");
    return fbank_launch(wave, ld_wave, n_samples, n_frames, B, t_max, window, twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift,
                        log2_nfft, snip_edges, remove_dc, n_mel, preemph, feats, dither, dither_seed,
                        reinterpret_cast<cudaStream_t>(stream), &mp);
}

/* the whole front end with MFCC features: the arguments of pk_frontend_fwd_noise_rir (null banks = no noise / no RIR), then the
 * MFCC epilogue's */
extern "C" int pk_frontend_fwd_mfcc(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                                    const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                                    int rctx, int stride, const float* window, const float* twiddle, const float* mel_w,
                                    const int* mel_lo, const int* mel_hi, int frame_len, int frame_shift, int log2_nfft,
                                    int snip_edges, int remove_dc, float preemph, int cmn, const float* offset, const float* scale,
                                    int f0, int fs, int t0, int ts, void* out, int out_dtype, short* wave_i16_out, void* workspace,
                                    long long workspace_bytes, int* err_flag, float dither, unsigned int dither_seed, void* stream,
                                    const short* noise, const int* noise_idx, const long long* noise_off, const double* snr,
                                    const double* noise_rms_db, const short* rir, const long long* rir_off, const int* rir_len,
                                    const int* rir_idx, int rir_max_len, const float* dct, int num_ceps, int use_energy,
                                    int raw_energy, float energy_floor, int htk_compat) {
    PK_CHECK_ARG(!noise || (noise_idx && noise_off && snr && noise_rms_db), "noise bank without its per-utterance draws");
    PK_CHECK_ARG(!rir || (rir_off && rir_len && rir_idx), "RIR bank without its offsets, lengths or per-utterance draws");
    const NoiseRirArgs nr{noise, noise_idx, noise_off, snr, noise_rms_db, rir, rir_off, rir_len, rir_idx, rir_max_len};
    const MfccParams mp{dct, num_ceps, use_energy ? 1 : 0, raw_energy ? 1 : 0, htk_compat ? 1 : 0, energy_floor};
    return frontend_launch(pcm, ld_pcm, n_samples, rate, new_len, target_db, n_frames, B, n_max, t_max, n_mel, lctx, rctx, stride, window,
                           twiddle, mel_w, mel_lo, mel_hi, frame_len, frame_shift, log2_nfft, snip_edges, remove_dc, preemph, cmn, offset,
                           scale, f0, fs, t0, ts, out, out_dtype, wave_i16_out, workspace, workspace_bytes, err_flag, dither, dither_seed,
                           stream, (noise || rir) ? &nr : nullptr, &mp);
}
