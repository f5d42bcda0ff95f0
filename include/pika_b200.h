/* pika_b200 -- C ABI of the H100-native RNN-Transducer hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference (tencent-ailab/pika) has
 * no FFI of its own: its hot path is Python calling torch / warp_rnnt / PyKaldi.  Each entry
 * point below names the reference call it replaces (paths relative to the reference root).
 * A maintainer binds these with ctypes (see INTEGRATION.md); pika_b200/_lib.py is that binding.
 *
 * Conventions: plain pointers and sizes only (no torch types); every function returns 0 on
 * success, <0 on error (pk_last_error() gives the message); device pointers unless noted;
 * functions never allocate device memory, never synchronise the stream, and are re-entrant per
 * stream.  `stream` is a cudaStream_t passed as void*.  dtype codes: 0 = float32, 1 = bfloat16.
 */
#ifndef PIKA_B200_H
#define PIKA_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PK_F32 0
#define PK_BF16 1

const char* pk_last_error(void);
int pk_version(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
long long pk_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Dense contractions on the Hopper tensor cores (wgmma, TMA-fed, bf16 x bf16 -> fp32).
 * Replaces every nn.Linear / nn.Conv2d(TDNN) / torch.matmul on the path:
 *   trainer/model/rnnt_tdnn_transformer.py:44-59,76-89 (fc_in, 9 TDNN convs, fc_out)
 *   trainer/model/modules/multi_headed_attn.py:180-182,207,223,233 (QKV, QK^T, PV, final_linear)
 *   trainer/model/modules/position_ffn.py:37-38 (w_1, w_2)
 *   trainer/model/transducer.py:56-61 (LSTM input/recurrent products), :108 (fc1, fc_gate, fc2)
 * and their autograd backward (dgrad / wgrad).
 *
 *   C[z][m][n] = epilogue( alpha * sum_p sum_kz sum_k A_p[z|kz][m + a_row_off_p][k] * B_p[z|kz][n + b_row_off_p][k] )
 *
 * Every operand is a 4-D strided view; dim[0] is the contiguous one.
 *   A, K-major : dim = (K, M, z2, z3)      A, MN-major: dim = (M, K, z2, z3)
 *   B, K-major : dim = (K, N, z2, z3)      B, MN-major: dim = (N, K, z2, z3)
 *   C          : dim = (N, M, zb0, zb1)
 * coordinates 2/3 of A and B are taken from (0 | zb0 | zb1 | kz) as chosen by *_sel.
 * Up to PK_GEMM_MAX_PAIRS (A_p, B_p) pairs accumulate into one tile: the 3 taps of a TDNN
 * layer (no im2col), and/or the 3 partial products of the split-bf16 "fp32-class" mode.
 */
#define PK_GEMM_MAX_PAIRS 9
#define PK_SEL_ZERO 0
#define PK_SEL_ZB0 1
#define PK_SEL_ZB1 2
#define PK_SEL_KZ 3
#define PK_ACT_NONE 0
#define PK_ACT_RELU 1
#define PK_AUX_NONE 0
#define PK_AUX_ADD 1      /* out += aux[m][n]                         (residual)            */
#define PK_AUX_MASK_NZ 2  /* out  = aux[m][n] != 0 ? out*aux_scale : 0 (ReLU/dropout backward) */

typedef struct {
    const void* ptr;    /* bf16 for A/B; bf16 or f32 for C */
    int64_t dim[4];     /* extents, dim[0] contiguous */
    int64_t stride[3];  /* strides of dims 1..3, in elements (multiples of 8 for bf16, 4 for f32) */
} pk_view4;

typedef struct {
    int n_pairs;
    pk_view4 a[PK_GEMM_MAX_PAIRS];
    pk_view4 b[PK_GEMM_MAX_PAIRS];
    int a_row_off[PK_GEMM_MAX_PAIRS]; /* added to the M (K-major) or K (MN-major) coordinate; may be negative */
    int b_row_off[PK_GEMM_MAX_PAIRS];
    int a_mn_major, b_mn_major;       /* 0 = K-major (reduction dim contiguous), 1 = MN-major */
    int a_sel2, a_sel3, b_sel2, b_sel3;
    int kz_count;                     /* extra (batched) reduction loop, >= 1 */
    pk_view4 c;
    int c_dtype;                      /* PK_F32 | PK_BF16 */
    int c_accumulate;                 /* 1: C += result (TMA reduce-add, f32 only) */
    /* epilogue, applied in this order */
    float alpha;
    const float* bias;                /* [N] or NULL */
    int act;
    float drop_p;                     /* 0 = off; keep-scale 1/(1-p) */
    uint32_t drop_seed;
    int aux_mode;
    const void* aux;                  /* same logical shape as C */
    int aux_dtype;
    int64_t aux_stride[3];            /* strides of (m, zb0, zb1) in elements */
    float aux_scale;
    int block_n;                      /* 0 = auto; else 64 | 128 | 256 */
    int k_splits;                     /* 0 = auto; 1 = off; >1 = split the reduction (plain f32 2-D C only) */
    float* row_lse;                   /* optional out [pk_gemm_row_lse_parts()][M][2] f32: per row and column group (max*log2(e),
                                         sum_j 2^(c_ij*log2(e) - max)) over the ROUNDED bf16 outputs -- the first pass of the fused
                                         log-softmax + RNN-T loss (pk_rnnt_loss_fwd_bwd_lse) computed while the logits tile is still in registers.
                                         Needs a 2-D bf16 C with N % 8 == 0, K-major operands, block_n 256. */
    const int* a_rows_dev;            /* optional device int32: only the first *a_rows_dev rows of A take part, read by the kernel, so
                                         the count needs no host synchronisation (the compacted joint gradient rows).  K-major A: C rows
                                         from *a_rows_dev on are undefined, whole BM-row tiles past it are skipped.  MN-major A (rows
                                         are K): the reduction stops at *a_rows_dev rounded up to 64, whose tail rows of A and B must
                                         hold zeros; the split-K splits share that shortened reduction.  One pair, kz_count 1, 2-D C. */
} pk_gemm_desc;

int pk_gemm_bf16(const pk_gemm_desc* desc, void* stream);
/* number of partials per row that pk_gemm_bf16 writes into row_lse for an [M, N] output with this block_n: one per N tile */
int pk_gemm_row_lse_parts(long long M, long long N, int block_n);

/* ------------------------------------------------------------------------------------------
 * RNN-T loss + gradient, fused with the log-softmax over V.
 * Replaces F.log_softmax (trainer/model/transducer.py:110-111) + warp_rnnt RNNTLoss.apply
 * (trainer/train_transducer_bmuf_otfaug.py:58,97-99; trainer/train_transducer_mbr_bmuf_otfaug.py:157-160)
 * and autograd's backward through both.
 *   logits  [B, T, U1, ldv] (first V of each row valid), dtype f32 | bf16, blank = 0
 *   labels  [B, ld_labels] int32; frame_lens, label_lens [B] int32 (T_n <= T, U_n <= U1-1)
 *   grad_scale [B] or NULL (dLoss/dcost_n, 1 when NULL)
 *   costs   [B] f32 = -log P(y_n | x_n)
 *   dlogits same shape/dtype as logits, may alias it (in place); NULL = loss only.
 *           Entries of padded nodes and of the row padding [V, ldv) are written as 0.
 *   dlogits_colsum [ldv] f32 or NULL: sum of dlogits over all (b,t,u) rows = the joint fc2 bias gradient,
 *           produced by the gradient pass itself (each thread owns fixed columns), so dlogits is not re-read.
 *           Deterministic: per-CTA partial rows are added in a fixed order (no atomics); when requested the workspace
 *           must hold pk_rnnt_loss_workspace_bytes + pk_rnnt_loss_colsum_workspace_bytes bytes.
 */
long long pk_rnnt_loss_workspace_bytes(int B, int T, int U1);
long long pk_rnnt_loss_colsum_workspace_bytes(int B, int T, int U1, int ldv);
int pk_rnnt_loss_fwd_bwd(const void* logits, int dtype, const int* labels, const int* frame_lens,
                         const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                         const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                         long long workspace_bytes, void* stream);
/* Same, with the first pass (row log-sum-exp) already done by the GEMM that produced the logits:
 * row_lse [n_parts][B*T*U1][2] as written through pk_gemm_desc.row_lse.  Saves one full read of the logits. */
int pk_rnnt_loss_fwd_bwd_lse(const void* logits, int dtype, const int* labels, const int* frame_lens,
                             const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                             const float* grad_scale, float* costs, void* dlogits, float* dlogits_colsum, void* workspace,
                             long long workspace_bytes, const float* row_lse, int n_parts, void* stream);
/* Same (row_lse may be NULL), bf16 only, with the gradient stored for the kept rows alone.  A row is skipped when |gb| + |gl| < 2^-136
 * for its blank / label occupancy terms: every entry of its bf16 gradient is then +-0, so it adds nothing to the fc2 GEMMs or the
 * bias gradient.  Outputs, all in device memory:
 *   row_map [B*T*U1] int32: the row's index among the kept rows (kept rows in (b, t, u) order), or -1
 *   row_count [1] int32: R' = the number of kept rows
 *   dz_c [B*T*U1, ldv]: rows [0, R') hold the kept rows' gradients (dlogits rebuilt as dlogits[r] = row_map[r] < 0 ? 0 : dz_c[row_map[r]]);
 *        rows [R', R' rounded up to 64) are written as zeros.  Must not alias logits.
 *   h_c [B*T*U1, H]: h_c[row_map[r]] = h[r] for the kept rows (the fc2 wgrad's other operand), zeros in the same tail rows as dz_c
 *   dlogits_colsum as above: the same sum in the same order as the dense form (a skipped row adds +-0 there).
 * H % 8 == 0, H <= 2048. */
int pk_rnnt_loss_fwd_bwd_compact(const void* logits, int dtype, const int* labels, const int* frame_lens,
                                 const int* label_lens, int B, int T, int U1, int V, int ldv, int ld_labels,
                                 const float* grad_scale, float* costs, void* dz_c, float* dlogits_colsum, void* workspace,
                                 long long workspace_bytes, const float* row_lse, int n_parts, const void* h, int H,
                                 void* h_c, int* row_map, int* row_count, void* stream);

/* The lattice pass alone, on log-prob tables the caller built (the simple and the pruned RNN-T losses below).
 *   lpb_skew, lpl_skew [B][T+U1-1][U1] f32: node (b, t, u) at ((b*(T+U1-1) + t+u)*U1 + u); lpb = log P(blank | t, u), lpl =
 *           log P(y_{u+1} | t, u) (read for u < U_b only).  -inf marks a node no path may use.  Every node t < T_b, u <= U_b is read.
 *   costs [B] = -log P(y | x) (+inf when no path has a finite score); gb, gl [B][T][U1] f32 = d cost / d lpb, d cost / d lpl (<= 0,
 *           times grad_scale[b] when grad_scale is not NULL; 0 at padded nodes).  -(gb + gl) is the node occupancy.
 *   workspace >= the size pk_rnnt_lattice_workspace writes to *bytes (the f64 alpha / beta). */
int pk_rnnt_lattice_workspace(int B, int T, int U1, long long* bytes);
int pk_rnnt_lattice(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew, const float* lpl_skew,
                    const float* grad_scale, float* costs, float* gb, float* gl, void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Pruned RNN-T loss (pika_b200/csrc/rnnt_pruned.cu, rnnt_loss.cu; DESIGN.md "Pruned RNN-T").
 * Simple joiner z[t,u] = am[t] + lm[u]; its normaliser N[t,u] = log(E_t . P_u) + max(am_t) + max(lm_u) with E = exp(am - rowmax),
 * P = exp(lm - rowmax), E.P^T a batched pk_gemm_bf16 product.  E.P below 2^-100 is clamped there (N stays finite; the clamped
 * node's normaliser is then constant in the gradient).
 *
 * pk_rnnt_simple_prep: src f32 rows (b, i < n_in) of [nb*n_in, ld_src] (V valid columns) -> hi (, lo: NULL or the bf16 residual)
 *   [nb*n_out, ld_out] bf16 = exp(src - rowmax), zero columns [V, ld_out) and zero rows i in [n_in, n_out); rmax [nb*n_in].
 * pk_rnnt_simple_tables: S [B*T, ld_s] f32 = E.P^T -> lpb_skew / lpl_skew (layout of pk_rnnt_lattice).
 * pk_rnnt_simple_w: gb, gl of that lattice -> W [B*T, ld_w] bf16 hi (, lo) = scale[b] * (-(gb + gl)) / S at the valid unclamped
 *   nodes, 0 elsewhere (including the columns [U1, ld_w)).  scale may be NULL (1).
 * pk_rnnt_simple_grad: axis 0 -> d am rows (b, t) [B*T, ldv]: exp(am - rmax) (.) G + scale * (sum_u gb at column 0, gl[t,u] at column
 *   y_{u+1}); axis 1 -> d lm rows (b, u) [B*U1, ldv]: the same with the sums over t.  G = W.P (axis 0) or W^T.E (axis 1), f32, row
 *   (b, i) at b*n_g + i, pitch ld_g.  One CTA per row; the blank / label terms are added by one thread in a fixed order.
 *   out_dtype PK_F32 | PK_BF16; columns [V, ldv) are written 0.  ldv <= 51200.
 * Smoothing (DESIGN.md "Pruned RNN-T"; lam_l = lm_only_scale, lam_a = am_only_scale, both >= 0 with lam_l + lam_a < 1, mu = 1 - both):
 * pk_rnnt_simple_smooth_stats: am [B*T, ldv], lm [B*U1, ldv] f32 (V valid columns) and their row maxes from pk_rnnt_simple_prep ->
 *   Nl [B*U1] = logsumexp_v lm[u], logq [ldv] = log(mean of softmax(lm[b, u]) over the batch's valid rows u <= U_b + 1e-10) (0 on
 *   the columns [V, ldv)), Na [B*T] = logsumexp_v (am[t] + logq).  Rows past T_b / U_b are written 0 and enter no sum; the unigram's
 *   column partials are summed per 64-row chunk, then in chunk order (no atomics).  workspace >= the size
 *   pk_rnnt_simple_smooth_stats_workspace writes to *bytes.
 * pk_rnnt_simple_tables_smooth: as pk_rnnt_simple_tables with lp = mu (z[k] - N) + lam_l (lm[u,k] - Nl[u]) + lam_a (am[t,k] + logq[k]
 *   - Na[t]) for k = 0 and k = y_{u+1}.
 * pk_rnnt_simple_grad_smooth: as pk_rnnt_simple_grad (G formed from W with the scale mu * scale[b]) with the blank / label terms
 *   weighted by scale[b] (mu + lam) and the row term scale[b] lam Gamma softmax(src [+ logq]), Gamma the row's summed occupancy;
 *   lam = lam_a with logq and lse = Na on axis 0, lam_l with lse = Nl on axis 1 (logq is not read there).
 * pk_rnnt_prune_bounds: occupancy gamma = -(ga + gb) (gb may be NULL) [B][T][U1] f32 -> bounds [B][T] int32 (DESIGN.md "Pruned RNN-T":
 *   window argmax in f64 with the smallest start on ties, clamp, running max, reverse pass; padded frames copy the last frame).
 *   An utterance with U_b > T_b (R-1) has no path inside the windows: its bounds are all -1 (the pruned loss is then +inf).
 * pk_joint_gate_pruned_fwd: h [B*T*R, H] row (b, t, r) = tanh(ex1[b,t] + py1[b,u]) * sigmoid(exg[b,t] + pyg[b,u]),
 *   u = min(max(bounds[b,t], 0) + r, U1 - 1).  ex [B*T, 2H], py [B*U1, 2H] as pk_joint_gate_fwd.
 * pk_joint_gate_pruned_bwd: dh [B*T*R, H] -> dex [B*T, 2H] (sum over r in order), dpy [B*U1, 2H] (sum over the frames whose window
 *   holds u, in frame order: one contiguous range because bounds are non-decreasing).  dh must be zero on the masked rows (u > U_b
 *   or t >= T_b), as pk_rnnt_pruned_loss writes it; rows whose u was clamped are not read.
 * pk_rnnt_pruned_loss: logits [B*T*R, ldv] (row (b, t, r) = node (t, bounds[b,t] + r)) -> costs [B], dlogits (may alias logits; NULL =
 *   costs only; masked rows and the padding columns written 0; needs ldv <= 8192, refused before any launch), dlogits_colsum [ldv]
 *   (NULL or the fc2 bias gradient, fixed-order sum).  Nodes outside the windows are -inf.  An utterance with bounds -1 gets cost +inf
 *   and zero dlogits rows.  row_lse: NULL or the producing GEMM's [n_parts][B*T*R][2] partials.
 *   workspace >= the size pk_rnnt_pruned_loss_workspace writes to *bytes. */
int pk_rnnt_simple_prep(const float* src, int ld_src, int V, int nb, int n_in, int n_out, void* hi, void* lo, int ld_out, float* rmax,
                        void* stream);
int pk_rnnt_simple_tables(const float* am, const float* lm, int ldv, const float* am_max, const float* lm_max, const float* S, int ld_s,
                          const int* labels, int ld_labels, const int* frame_lens, const int* label_lens, int B, int T, int U1,
                          float* lpb_skew, float* lpl_skew, void* stream);
int pk_rnnt_simple_w(const float* gb, const float* gl, const float* S, int ld_s, const int* frame_lens, const int* label_lens,
                     const float* scale, int B, int T, int U1, void* w_hi, void* w_lo, int ld_w, void* stream);
int pk_rnnt_simple_grad(const float* src, int ldv, int V, const float* rmax, const float* G, int ld_g, int n_g, int axis, const float* gb,
                        const float* gl, const int* labels, int ld_labels, const int* frame_lens, const int* label_lens, const float* scale,
                        int B, int T, int U1, void* out, int out_dtype, void* stream);
int pk_rnnt_simple_smooth_stats_workspace(int B, int U1, int ldv, long long* bytes);
int pk_rnnt_simple_smooth_stats(const float* am, const float* lm, int ldv, int V, const float* am_max, const float* lm_max,
                                const int* frame_lens, const int* label_lens, int B, int T, int U1, float* Nl, float* logq, float* Na,
                                void* workspace, long long workspace_bytes, void* stream);
int pk_rnnt_simple_tables_smooth(const float* am, const float* lm, int ldv, const float* am_max, const float* lm_max, const float* S,
                                 int ld_s, const int* labels, int ld_labels, const int* frame_lens, const int* label_lens, int B, int T,
                                 int U1, const float* Nl, const float* logq, const float* Na, float lm_only_scale, float am_only_scale,
                                 float* lpb_skew, float* lpl_skew, void* stream);
int pk_rnnt_simple_grad_smooth(const float* src, int ldv, int V, const float* rmax, const float* G, int ld_g, int n_g, int axis,
                               const float* gb, const float* gl, const int* labels, int ld_labels, const int* frame_lens,
                               const int* label_lens, const float* scale, const float* logq, const float* lse, float lm_only_scale,
                               float am_only_scale, int B, int T, int U1, void* out, int out_dtype, void* stream);
int pk_rnnt_prune_bounds(const float* ga, const float* gb, const int* frame_lens, const int* label_lens, int B, int T, int U1, int R,
                         int* bounds, void* stream);
int pk_joint_gate_pruned_fwd(const void* ex, const void* py, const int* bounds, void* h, int dtype, int B, int T, int U1, int R, int H,
                             void* stream);
int pk_joint_gate_pruned_bwd(const void* ex, const void* py, const int* bounds, const void* dh, void* dex, void* dpy, int dtype, int B,
                             int T, int U1, int R, int H, void* stream);
int pk_rnnt_pruned_loss_workspace(int B, int T, int U1, int R, int ldv, long long* bytes);
int pk_rnnt_pruned_loss(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, const int* bounds,
                        int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* grad_scale, float* costs, void* dlogits,
                        float* dlogits_colsum, void* workspace, long long workspace_bytes, const float* row_lse, int n_parts,
                        void* stream);

/* ------------------------------------------------------------------------------------------
 * RNN-T forced alignment (pika_b200/csrc/rnnt_loss.cu; DESIGN.md "Forced alignment").  Tables in the layout of pk_rnnt_lattice.
 * pk_rnnt_tables: the dense loss's first pass alone: logits [B, T, U1, ldv] (as pk_rnnt_loss_fwd_bwd) -> lse [B*T*U1] f32 (the row
 *   log-sum-exp), lpb_skew, lpl_skew.  row_lse: NULL (the logits are streamed) or the producing GEMM's [n_parts][B*T*U1][2] partials.
 *   Nodes t >= T_b or u > U_b are not written.  No gradient buffer is touched.
 * pk_rnnt_pruned_tables: pk_rnnt_pruned_loss's tables alone: logits [B*T*R, ldv] + bounds -> lse [B*T*R], lpb_skew / lpl_skew with -inf
 *   outside each frame's window of R label positions.
 * pk_rnnt_lattice_costs: pk_rnnt_lattice without gb / gl: costs [B] = -log P(y | x) only (same workspace).
 * pk_rnnt_viterbi: best path through the lattice, f64 max-plus: delta(0,0) = 0, delta(t,u) = max(delta(t-1,u) + lpb(t-1,u),
 *   delta(t,u-1) + lpl(t,u-1)); the label arc is taken only when strictly greater (ties and -inf on both arcs: blank).
 *   score [B] f32 = delta(T_b-1, U_b) + lpb(T_b-1, U_b), -inf when no path has a finite score (or T_b = 0).
 *   emit_frames [B][ld_emit] int32 (ld_emit >= U1 - 1): entry u-1 = the frame t of the best path's label arc (t, u-1) -> (t, u) for
 *   u = 1 .. U_b, non-decreasing in u; -1 from U_b on, and everywhere when score is -inf.
 *   workspace >= the size pk_rnnt_viterbi_workspace writes to *bytes; on return it holds the decisions: u32 words
 *   [B][T+U1-1][ceil(U1/32)], bit u % 32 of word (b, t+u, u / 32) = 1 when node (t, u) of a valid utterance came in by its label arc
 *   (words whose first u is past U_b are not written).  U1 <= 2048; one CTA per utterance, no atomics: deterministic. */
int pk_rnnt_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, int B, int T, int U1,
                   int V, int ldv, int ld_labels, const float* row_lse, int n_parts, float* lse, float* lpb_skew, float* lpl_skew,
                   void* stream);
int pk_rnnt_pruned_tables(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                          const int* bounds, int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* row_lse, int n_parts,
                          float* lse, float* lpb_skew, float* lpl_skew, void* stream);
int pk_rnnt_lattice_costs(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew, const float* lpl_skew,
                          float* costs, void* workspace, long long workspace_bytes, void* stream);
int pk_rnnt_viterbi_workspace(int B, int T, int U1, long long* bytes);
int pk_rnnt_viterbi(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew, const float* lpl_skew,
                    float* score, int* emit_frames, int ld_emit, void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * RNN-T emission regularisation (pika_b200/csrc/rnnt_loss.cu; DESIGN.md "FastEmit and delay penalty").  Each *_reg entry point is
 * the entry point of the same name without the suffix, with two more arguments, both finite and >= 0 (refused before any launch):
 *   delay_penalty lambda_d: every label arc (t, u) -> (t, u+1) of utterance b has lambda_d * ((T_b - 1)/2 - t) added to its log-prob,
 *           in f64 where the lattice reads it (the tables are not changed).  costs are the penalised -log P and gb / gl its exact
 *           gradient (the term does not depend on the logits).
 *   fastemit_lambda lambda_f: the label coefficient gl is multiplied by 1 + lambda_f (FastEmit).  The cost is unchanged, so with
 *           lambda_f > 0 the gradient is not the gradient of the returned cost.
 * With both 0 the outputs and launches are those of the plain entry point. */
int pk_rnnt_loss_fwd_bwd_reg(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, int B, int T,
                             int U1, int V, int ldv, int ld_labels, const float* grad_scale, float* costs, void* dlogits,
                             float* dlogits_colsum, void* workspace, long long workspace_bytes, float fastemit_lambda, float delay_penalty,
                             void* stream);
int pk_rnnt_loss_fwd_bwd_lse_reg(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, int B,
                                 int T, int U1, int V, int ldv, int ld_labels, const float* grad_scale, float* costs, void* dlogits,
                                 float* dlogits_colsum, void* workspace, long long workspace_bytes, const float* row_lse, int n_parts,
                                 float fastemit_lambda, float delay_penalty, void* stream);
int pk_rnnt_loss_fwd_bwd_compact_reg(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens, int B,
                                     int T, int U1, int V, int ldv, int ld_labels, const float* grad_scale, float* costs, void* dz_c,
                                     float* dlogits_colsum, void* workspace, long long workspace_bytes, const float* row_lse, int n_parts,
                                     const void* h, int H, void* h_c, int* row_map, int* row_count, float fastemit_lambda,
                                     float delay_penalty, void* stream);
int pk_rnnt_lattice_reg(const int* frame_lens, const int* label_lens, int B, int T, int U1, const float* lpb_skew, const float* lpl_skew,
                        const float* grad_scale, float* costs, float* gb, float* gl, void* workspace, long long workspace_bytes,
                        float fastemit_lambda, float delay_penalty, void* stream);
int pk_rnnt_pruned_loss_reg(const void* logits, int dtype, const int* labels, const int* frame_lens, const int* label_lens,
                            const int* bounds, int B, int T, int U1, int R, int V, int ldv, int ld_labels, const float* grad_scale,
                            float* costs, void* dlogits, float* dlogits_colsum, void* workspace, long long workspace_bytes,
                            const float* row_lse, int n_parts, float fastemit_lambda, float delay_penalty, void* stream);

/* ------------------------------------------------------------------------------------------
 * Memory-bound layers around the GEMMs (pika_b200/csrc/elementwise.cu).  `dtype` is the
 * activation type (PK_BF16 production, PK_F32 fp32-class parity mode); statistics are f32.
 */
/* bf16 (hi) and optional residual (lo) copies of an f32/bf16 matrix, zero-padded to cols_pad:
 * weight/activation staging for pk_gemm_bf16 (replaces the implicit casts of torch autocast-free fp32). */
int pk_cast_split(const void* src, int src_dtype, long long ld_src, void* hi, void* lo, long long ld_dst,
                  long long rows, int cols, int cols_pad, float scale, void* stream);
/* Fused unmasked multi-head self-attention, head dim 64, bf16 (pika_b200/csrc/attention_tc.cu):
 *   O = dropout(softmax(alpha * Q K^T)) V  per (batch, head)   -- MultiHeadedAttention.forward,
 *   trainer/model/modules/multi_headed_attn.py:199-223 (scale, softmax, dropout, context) and its autograd backward,
 * without materialising the [B, heads, T, T] score / probability tensors.
 *   q, k, v: element (b, t, h, d) at ptr[(b*T + t)*ld_qkv + h*64 + d]  (three column blocks of a fused [B,T,3D] projection)
 *   out / dout [B, T, heads*64] with row strides ld_out / ld_dout;  lse [B*heads][pk_attention_lse_stride(T)] f32: the natural-log
 *   row log-sum-exp of the scaled scores, entry t of (b, h) at lse[(b*heads + h)*pk_attention_lse_stride(T) + t], saved for the backward
 *   dq, dk, dv: same addressing with row stride ld_dqkv;  dsum_ws: [B*heads][pk_attention_lse_stride(T)] f32 scratch
 *   The padding t in [T, pk_attention_lse_stride(T)) of lse and dsum_ws is written by the kernels themselves (lse by the forward,
 *   dsum_ws by the backward), so neither buffer needs initialising; the backward takes lse as the forward wrote it.
 * Dropout masks are the same counter-based masks as pk_softmax_fwd/bwd for equal (drop_p, seed): row (b*heads + h)*T + t.
 * pk_attention_fwd / pk_attention_bwd draw the mask from seed in every kernel.  pk_attention_fwd_bits also writes every keep decision
 * as one bit into keep_bits, and pk_attention_bwd_bits reads those bits instead of hashing (so it takes no seed) -- the cheaper pair
 * for a forward whose backward follows.  keep_bits is caller-allocated, pk_attention_keep_bits_bytes(B, T, heads) bytes, 16-byte
 * aligned, needs no initialising, and may be NULL only when drop_p == 0.  Layout, with n = 2 * ceil(T / 128) blocks of 64 along each axis:
 *   words [B*heads][n query blocks][n key blocks][128] (uint32); in block (qb, kb) the decision for query qb*64 + r, key kb*64 + c
 *   is bit ((r >> 3) & 1) * 16 + (c >> 3) * 2 + (c & 1) of word (r >> 4) * 32 + ((c & 7) >> 1) * 8 + (r & 7).
 * That is the wgmma accumulator layout of the 64 x 64 score block: the thread that holds (r, c) in the forward and dQ kernels owns
 * the whole word, and the dK/dV kernel, which holds the transposed block, finds its 32 decisions in four pairs of adjacent words.
 * Blocks beyond the sequence (query or key >= T) are never read for a decision that reaches an output. */
/* row pitch of lse / dsum_ws: T rounded up to a multiple of 64 */
int pk_attention_lse_stride(int T);
/* bytes of the keep-bit buffer: B * heads * (2 * ceil(T / 128))^2 * 512 */
long long pk_attention_keep_bits_bytes(int B, int T, int heads);
int pk_attention_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                     int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, void* stream);
int pk_attention_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                     const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                     long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, void* stream);
int pk_attention_fwd_bits(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                          int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, uint32_t* keep_bits, void* stream);
int pk_attention_bwd_bits(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                          const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                          long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, const uint32_t* keep_bits,
                          void* stream);
/* Chunk-masked (streaming) self-attention, keep-bits form (DESIGN.md "Chunked attention").  Frame t lies in chunk
 * (t + chunk_off) / chunk_len; query i sees key j iff chunk(i) - left_chunks <= chunk(j) <= chunk(i), with no lower limit when
 * left_chunks = -1.  A frame always sees itself.  Arguments otherwise as pk_attention_fwd_bits / pk_attention_bwd_bits, with the same
 * dropout decisions for every pair; keep_bits may be NULL only when drop_p == 0.  The kernels skip every 64-wide key tile (the dK/dV
 * kernel: query tile) that no row of the 128-row block sees, and never write or read the keep bits of a skipped tile.  The lse padding
 * entries are written as without the mask.  A mask that lets every query see every key runs the unmasked kernels.
 * Refused before any launch: chunk_len < 1, chunk_off < 0, left_chunks < -1. */
int pk_attention_fwd_chunk(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out, float* lse,
                           int B, int T, int heads, int dh, float alpha, float drop_p, uint32_t seed, uint32_t* keep_bits,
                           int chunk_len, int chunk_off, int left_chunks, void* stream);
int pk_attention_bwd_chunk(const void* q, const void* k, const void* v, long long ld_qkv, const void* out, long long ld_out,
                           const void* dout, long long ld_dout, const float* lse, float* dsum_ws, void* dq, void* dk, void* dv,
                           long long ld_dqkv, int B, int T, int heads, int dh, float alpha, float drop_p, const uint32_t* keep_bits,
                           int chunk_len, int chunk_off, int left_chunks, void* stream);
/* 1 when that mask lets every query of a T-frame sequence see every key, 0 when it does not, -1 on bad arguments (a pure host function) */
int pk_attention_chunk_admits_all(int T, int chunk_len, int chunk_off, int left_chunks);
/* nn.BatchNorm1d over rows [rows, C] (trainer/model/rnnt_tdnn_transformer.py:41,58-59,69,76-82,85):
 * train: batch statistics incl. padded frames, running stats updated with the given momentum (unbiased variance); eval: running
 * stats.  stats_ws: pk_colstats_ws_floats(C) + 2*C floats scratch.  mean/rstd [C] are saved for the backward.
 * x, y, stats_ws (and dy, dx, ws of the backward, x of pk_colsum) must be 16-byte aligned. */
long long pk_colstats_ws_floats(int C);
int pk_bn_fwd(const void* x, void* y, int dtype, long long rows, int C, const float* w, const float* b, float eps,
              int train, float momentum, float* run_mean, float* run_var, float* mean, float* rstd, float* stats_ws,
              void* stream);
/* BN backward; relu_mask=1 additionally multiplies by (x > 0): x is the BN input = ReLU output, so the
 * result is the gradient w.r.t. the pre-ReLU TDNN/Linear output.  dw, db [C] are overwritten. */
int pk_bn_bwd(const void* dy, const void* x, void* dx, int dtype, long long rows, int C, const float* w,
              const float* mean, const float* rstd, int train, int relu_mask, float* dw, float* db, float* ws /* pk_colstats_ws_floats(C) */,
              void* stream);
/* out[c] = sum_r x[r,c]  (bias gradients); ws: pk_colstats_ws_floats(C) floats */
int pk_colsum(const void* x, int dtype, long long rows, int C, float* out, float* ws, void* stream);
/* nn.LayerNorm(C, eps=1e-6) (trainer/model/modules/transformer.py:82, position_ffn.py:21) */
int pk_layernorm_fwd(const void* x, void* y, int dtype, long long rows, int C, const float* w, const float* b, float eps,
                     float* mean, float* rstd, void* stream);
int pk_layernorm_bwd(const void* dy, const void* x, void* dx, int dtype, long long rows, int C, const float* w,
                     const float* mean, const float* rstd, float* dw, float* db, void* stream);
/* attention softmax over keys + dropout on the probabilities
 * (trainer/model/modules/multi_headed_attn.py:220-221): S f32 [rows, ld_s] -> P, Pd=dropout(P) [rows, ld_p] */
int pk_softmax_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                   float drop_p, uint32_t seed, void* stream);
/* masked forward (transformer prediction net, trainer/model/rnnt_conv_transformer_lm.py:66-70 + modules/multi_headed_attn.py:214-216):
 * rows = sequences * heads * q_len; key c of query i = row % q_len is dropped when (causal && c > i) or key_pad[sequence][c] != 0
 * (key_pad: uint8 [sequences][n] or NULL).  The backward is pk_softmax_bwd (a dropped key has P = 0). */
int pk_softmax_masked_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                          int q_len, int heads, int causal, const uint8_t* key_pad, float drop_p, uint32_t seed, void* stream);
/* chunk-masked self-attention forward (the chunk mask of pk_attention_fwd_chunk): rows = sequences * heads * n, query i = row % n keeps
 * the keys its chunk allows (always i itself).  The backward is pk_softmax_bwd.  Bad chunk arguments are refused before any launch. */
int pk_softmax_chunk_fwd(const float* S, long long ld_s, void* P, void* Pd, int dtype, long long ld_p, long long rows, int n,
                         int chunk_len, int chunk_off, int left_chunks, float drop_p, uint32_t seed, void* stream);
int pk_softmax_bwd(const float* dPd, long long ld_d, const void* P, long long ld_p, void* dS, int dtype, long long rows,
                   int n, float drop_p, uint32_t seed, void* stream);
/* Relative-position self-attention (Shaw et al.; trainer/model/modules/multi_headed_attn.py:9-41,186-229), max_rel = m > 0:
 *   scores_ij = alpha q_i.k_j + alpha q_i.R[b(i,j)],  out_i = sum_j Pd_ij v_j + sum_j Pd_ij R[b(i,j)],  b(i,j) = clamp(j-i, -m, m) + m
 * with R the [2m+1, dh] table (key and value relations alike).  The GEMMs around these kernels form QR = alpha Q R^T and
 * G = dO R^T; the kernels gather them along the band and reduce P / dS back onto the 2m+1 buckets.
 * Rows of S / P / dPd / dS are (sequence, head, query i) as for pk_softmax_masked_fwd, with q_len = n (self-attention).  Rows of
 * QR, Pb, G, dSb ([sequences * n * heads, ld_r] f32) are token-major: (sequence, query i, head).
 *   fwd: P = softmax(mask(S + QR[b])), Pd = dropout(P) as pk_softmax_masked_fwd (causal and key_pad optional here);
 *        Pb[., r] = sum over keys j with b(i,j) = r of Pd (as stored).
 *   bwd: dS = softmax_bwd(dPd + G[b]) as pk_softmax_bwd;  dSb[., r] = sum over keys j with b(i,j) = r of dS (as stored).
 * Every entry of Pb / dSb is written (0 for buckets no key reaches and for the padding [2m+1, ld_r)).
 * Limits: n <= ld_p <= 2048 (the row lives in one warp's registers), ld_s / ld_d >= ld_p, pitches multiples of 8;
 *         1 <= m <= 1024, ld_r >= 2m+1 and a multiple of 8. */
#define PK_RELPOS_MAX 1024
int pk_softmax_masked_relpos_fwd(const float* S, long long ld_s, const float* QR, long long ld_r, void* P, void* Pd, int dtype,
                                 long long ld_p, long long rows, int n, int q_len, int heads, int causal, const uint8_t* key_pad,
                                 int max_rel, float* Pb, float drop_p, uint32_t seed, void* stream);
int pk_softmax_relpos_bwd(const float* dPd, long long ld_d, const float* G, long long ld_r, const void* P, long long ld_p, void* dS,
                          int dtype, long long rows, int n, int q_len, int heads, int max_rel, float* dSb, float drop_p,
                          uint32_t seed, void* stream);
/* nn.Dropout with the counter-based RNG shared with the GEMM epilogue; mask_nz: dx = dy * (y != 0) * scale */
int pk_dropout(const void* x, void* y, int dtype, long long n, float p, uint32_t seed, void* stream);
int pk_mask_nz(const void* dy, const void* y, void* dx, int dtype, long long n, float scale, void* stream);
int pk_add(const void* a, const void* b, void* o, int dtype, long long n, void* stream);
/* F.log_softmax(scale * x) rows -> f32 (trainer/model/transducer.py:110-111; decoder/transducer_decoder.py:177) */
int pk_log_softmax(const void* x, int dtype, long long ld, float* y, long long rows, int n, float scale, void* stream);
/* gated joint, factored: h[b,t,u,:] = tanh(e1[b,t]+p1[b,u]) * sigmoid(eg[b,t]+pg[b,u])
 * (trainer/model/transducer.py:102-108 without materialising the 2H-wide concat).
 * ex [B*T, 2H], py [B*U1, 2H] = the x / y halves of fc1 | fc_gate applied to encoder / prediction outputs. */
/* h has row pitch ld_h = H or H+8; with H+8 the pad columns are written as (1,0,..,0) so that the fc2 bias gradient
 * falls out of the fc2 wgrad GEMM as one extra column */
int pk_joint_gate_fwd(const void* ex, const void* py, void* h, int dtype, int B, int T, int U1, int H, int ld_h, void* stream);
/* dh_map: NULL (dh is [B*T*U1, H]) or a row map of pk_rnnt_loss_fwd_bwd_compact: the dh row of joint row r is dh[dh_map[r]], zeros
 * when dh_map[r] < 0 (dh then holds the compacted rows). */
int pk_joint_gate_bwd(const void* ex, const void* py, const void* dh, const int* dh_map, void* dex, void* dpy, int dtype, int B, int T,
                      int U1, int H, void* stream);
/* one LSTM time step, pointwise part (nn.LSTM, gate order i,f,g,o; trainer/model/transducer.py:56-61) */
int pk_lstm_cell_fwd(const float* gx, long long ld_gx, const float* gh, long long ld_gh, const float* c_prev, float* c_out,
                     void* h_out, int dtype, long long ld_h, float* gates_save, int B, int H, void* stream);
int pk_lstm_cell_bwd(const void* dh_out, long long ld_dho, const float* dh_rec, const float* dc_next, const float* gates,
                     const float* c, const float* c_prev, void* dgates, int dtype, float* dc_prev, int B, int H, void* stream);
/* nn.Embedding (trainer/model/transducer.py:52-53,94); rows padded to ld_out; padding_idx gets no gradient */
int pk_embedding_fwd(const long long* idx, const float* table, int E, void* out, int dtype, int ld_out, long long n, void* stream);
int pk_embedding_bwd(const long long* idx, const void* dout, int dtype, int ld, int E, float* dtable, long long n,
                     long long padding_idx, void* stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser / BMUF on the flat fp32 parameter vector (pika_b200/csrc/optim.cu).
 *   pk_absmax + pk_sgd_nesterov_clip: clip_grad_norm_(params, max_norm, inf) + optim.SGD(nesterov).step()
 *                                     (trainer/train_transducer_bmuf_otfaug.py:53-55,105-110)
 *   pk_bmuf_delta / pk_bmuf_update  : BmufTrainer.update_and_sync (trainer/bmuf.py:76-100); the sum over
 *                                     ranks between the two is an NCCL all-reduce issued by the host side.
 */
int pk_absmax(const float* x, long long n, float* out, int* nan_flag, void* stream);
/* nan_flag (may be NULL): the flag pk_absmax raised; when set the clip coefficient is NaN, as torch's clip_grad_norm_(inf) gives */
int pk_sgd_nesterov_clip(float* p, const float* g, float* buf, long long n, float lr, float momentum, float max_norm,
                         const float* absmax, const int* nan_flag, int first, void* stream);
int pk_bmuf_delta(const float* glob, const float* local, float* delta, long long n, void* stream);
int pk_bmuf_update(float* glob, float* local, float* delta_prev, const float* delta_sum, long long n, int world,
                   float block_momentum, float block_lr, void* stream);
/* pk_absmax + pk_adam_clip: clip_grad_norm_(params, max_norm, inf) + optim.Adam(lr, betas, eps, weight_decay=0,
 * amsgrad=False).step() (trainer/bmuf.py:204,215 -- the local optimiser of BmufAdamTrainer) over (p, g, exp_avg, exp_avg_sq).
 * The clip and its NaN rule are pk_sgd_nesterov_clip's (max_norm <= 0: no clip).  The caller forms the bias corrections
 * 1 - beta1^step and sqrt(1 - beta2^step) in double; step may be fractional after a BMUF-Adam sync (trainer/bmuf.py:311).
 * Element formula as torch's CUDA Adam: m.lerp_(g, 1-beta1); v = beta2*v + (1-beta2)*g*g;
 * p -= (lr/bias_correction1) * m / (sqrt(v)/bias_correction2_sqrt + eps).
 * p_out2 (may be NULL): also receives the new p -- BlockAdamTrainer's copy of the global vector into the model
 * (trainer/bmuf.py:163-166) in the same pass. */
int pk_adam_clip(float* p, const float* g, float* exp_avg, float* exp_avg_sq, float* p_out2, long long n, double lr,
                 double beta1, double beta2, double eps, double bias_correction1, double bias_correction2_sqrt,
                 float max_norm, const float* absmax, const int* nan_flag, void* stream);
/* BmufAdamTrainer.update_and_sync (trainer/bmuf.py:273-321), the master update replicated on every rank after an all-reduce.
 * msg = [delta_sum; exp_avg_sum; exp_avg_sq_sum] (3n floats, the summed pk_bmuf_delta output and local moments).  Updates the
 * global parameters glob and delta_prev (block momentum, as pk_bmuf_update), the filtered global moments exp_avg_g /
 * exp_avg_sq_g, writes local := glob, and overwrites msg's two moment slots with the new local moments.  beta1_tau = beta1^tau,
 * beta1_rho = beta1^(rho*block_momentum) (likewise beta2), formed by the caller in double; tau = sync_period and rho is the
 * already-updated block-momentum sum of :273. */
int pk_bmuf_adam_update(float* glob, float* local, float* delta_prev, float* exp_avg_g, float* exp_avg_sq_g, float* msg,
                        long long n, int world, double block_momentum, double block_lr, double beta1_tau, double beta1_rho,
                        double beta2_tau, double beta2_rho, void* stream);

/* ------------------------------------------------------------------------------------------
 * On-the-fly front end (pika_b200/csrc/frontend.cu): int16 PCM -> speed perturbation + RMS gain +
 * int16 re-quantisation -> Kaldi fbank -> splice -> last-frame padding -> CMN/CMVN -> SpecAugment.
 * Replaces loader/audio.py (AudioSegment.change_speed/normalize/_convert_*), the PyKaldi
 * Fbank.compute_features call and splice() in loader/otf_utt_loader.py:28-46,195-201,218-234,262-270,
 * and trainer/train_transducer_bmuf_otfaug.py:86-93 + utils/spec_augment.py:10-20.
 *   pcm [B, ld_pcm] int16; n_samples, new_len (= int(n/rate)) [B] int32
 *   n_frames [B] int32: fbank frames of new_len samples; snip_edges: 0 if new_len < frame_len, else 1+(new_len-frame_len)/frame_shift;
 *     otherwise (new_len + frame_shift/2) / frame_shift, frame t starting at t*frame_shift + frame_shift/2 - frame_len/2 with the
 *     samples outside [0, new_len) reflected about the edges (Kaldi's ExtractWindow).  Precondition the host cannot check (the
 *     lengths live on the device): with snip_edges = 0, new_len[b] >= 1 wherever n_frames[b] > 0 -- reflection about an empty
 *     signal never ends.  The same holds for n_samples of pk_fbank / pk_mfcc.
 *   t_max: output rows; stride: output row t is spliced fbank frame min(t, ceil(n_frames/stride)-1)*stride, i.e.
 *     splice(feats)[::stride] padded with its last row.  Workspace queries take t_max*stride, the fbank frames held in between.
 *   rate, target_db [B] f32 (host-drawn, as the reference draws them in the loader thread)
 *   window [frame_len], twiddle [N/2 x (re,im)] = exp(-2 pi i k / N), mel_w [n_mel, N/2], mel_lo/hi [n_mel]: host-built tables for
 *     the FFT size N = 2^log2_nfft, 128 <= N <= 2048, 1 <= frame_len <= N; n_max >= frame_len when snip_edges is set
 *   remove_dc: subtract each window's mean (Kaldi --remove-dc-offset); preemph: --preemphasis-coefficient
 *   offset/scale [D] CMVN (NULL = off); cmn: subtract the per-utterance mean over the PADDED time axis, summed in a fixed order
 *     (row order within blocks of 64 rows, then block order), so that repeated runs give the same bits
 *   (f0,fs,t0,ts): SpecAugment freq/time mask start and span (span 0 = off), shared by the batch
 *   out [B, t_max, D] f32|bf16; wave_i16_out [B, n_max] optional copy of the augmented samples
 *   err_flag: set to 1 if a gain above 300 dB was requested (the reference raises ValueError)
 *   dither, dither_seed: FbankOptions.dither (egs/fbank.conf: dither=1): dither * N(0,1) added to every sample of every extracted
 *   window, as Kaldi's Dither() does; the draws come from a counter-based generator keyed by (utterance, frame, sample, seed) --
 *   Kaldi's own RNG stream is not reproduced.  0 = off (bit-reproducible features, what the parity tests use).
 */
long long pk_frontend_workspace_bytes(int B, int n_max, int t_max, int n_mel, int D);
int pk_frontend_fwd(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                    const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                    int rctx, int stride, const float* window, const float* twiddle, const float* mel_w, const int* mel_lo,
                    const int* mel_hi, int frame_len, int frame_shift, int log2_nfft, int snip_edges, int remove_dc,
                    float preemph, int cmn, const float* offset, const float* scale, int f0, int fs,
                    int t0, int ts, void* out, int out_dtype, short* wave_i16_out, void* workspace,
                    long long workspace_bytes, int* err_flag, float dither, unsigned int dither_seed, void* stream);
/* pk_fbank: the fbank stage alone (no stride); n_samples [B] (the reflected edges' bound) may be NULL when snip_edges is set */
int pk_fbank(const float* wave, long long ld_wave, const int* n_samples, const int* n_frames, int B, int t_max, int n_mel,
             const float* window, const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi, int frame_len,
             int frame_shift, int log2_nfft, int snip_edges, int remove_dc, float preemph, float* feats, float dither,
             unsigned int dither_seed, void* stream);

/* Front end with on-the-fly noise and reverberation (loader/audio.py:426-513 AudioSegment.add_noise / convolve_and_normalize,
 * loader/otf_utt_loader.py:224-228), per utterance: speed -> normalize(target_db) -> add_noise -> convolve_and_normalize -> int16
 * -> fbank ...  Arguments up to `stream` are those of pk_frontend_fwd; then
 *   noise        int16 bank of concatenated noise segments (device), or null for no noise
 *   noise_idx    [B] int32 segment of each utterance; noise_off [B] int64 ABSOLUTE bank offset of the utterance's first noise
 *                sample (segment start + drawn offset; new_len[b] samples are read); snr [B] f64 dB
 *   noise_rms_db [n_noise] f64: rms_db of each whole segment (float32 samples, as AudioSegment.rms_db)
 *   rir          int16 bank of concatenated RIRs (device), or null for no reverberation
 *   rir_off      [n_rir] int64 start, rir_len [n_rir] int32 length (>= 1), rir_idx [B] int32 RIR of each utterance
 *   rir_max_len  host-side bound >= every rir_len[rir_idx[b]], in [1, 65536] (pass 1 without RIRs); sets the FFT block length.
 *                Precondition the host cannot check (the lengths live on the device): a drawn RIR longer than rir_max_len is
 *                silently truncated to its first ceil(rir_max_len / Lb) blocks of Lb samples
 * The convolution is fftconvolve(x, h, "same") in float64 (uniformly partitioned overlap-save); on the rate == 1.0 branch the
 * result is rounded to float32, like the reference's float32 samples.  err_flag also reports a renormalisation gain above 300 dB.
 * Workspace: pk_frontend_noise_rir_workspace_bytes (< 0 when rir_max_len is outside [1, 65536]; no device access). */
long long pk_frontend_noise_rir_workspace_bytes(int B, int n_max, int t_max, int n_mel, int D, int rir_max_len);
int pk_frontend_fwd_noise_rir(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                              const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                              int rctx, int stride, const float* window, const float* twiddle, const float* mel_w,
                              const int* mel_lo, const int* mel_hi, int frame_len, int frame_shift, int log2_nfft, int snip_edges,
                              int remove_dc, float preemph, int cmn, const float* offset, const float* scale, int f0, int fs,
                              int t0, int ts, void* out, int out_dtype, short* wave_i16_out, void* workspace,
                              long long workspace_bytes, int* err_flag, float dither, unsigned int dither_seed, void* stream,
                              const short* noise, const int* noise_idx, const long long* noise_off, const double* snr,
                              const double* noise_rms_db, const short* rir, const long long* rir_off, const int* rir_len,
                              const int* rir_idx, int rir_max_len);

/* Kaldi MFCC (feat/feature-mfcc.cc MfccComputer::Compute) in place of fbank: the same frames, window, FFT and mel banks, then per frame
 * c = dct . log(max(mel, FLT_EPSILON)), and
 *   dct          [n_mel, num_ceps] f32: the first num_ceps rows of the orthonormal DCT-II of size n_mel, each times its lifter
 *                coefficient 1 + Q/2 sin(pi k / Q) (Q = --cepstral-lifter, none when 0), stored transposed; 1 <= num_ceps <= n_mel
 *   use_energy   c0 <- log(max(E, FLT_EPSILON)), raised to log(energy_floor) when energy_floor > 0; E is the sum of squares of the
 *                window after dither and DC removal (raw_energy) or of the windowed, pre-emphasised frame (otherwise)
 *   htk_compat   c0 (or the energy) moves to the last column; without use_energy it is multiplied by sqrt(2)
 * Features are num_ceps wide: the splice, CMN/CMVN and SpecAugment stages and the workspace queries take num_ceps where the fbank
 * entry points take n_mel (D = num_ceps * (lctx + 1 + rctx)).
 * pk_mfcc: arguments up to `stream` are those of pk_fbank; feats [B, t_max, num_ceps].
 * pk_frontend_fwd_mfcc: arguments up to `rir_max_len` are those of pk_frontend_fwd_noise_rir, whose banks may both be null (then the
 * sequence of pk_frontend_fwd runs, and pk_frontend_workspace_bytes suffices). */
int pk_mfcc(const float* wave, long long ld_wave, const int* n_samples, const int* n_frames, int B, int t_max, int n_mel,
            const float* window, const float* twiddle, const float* mel_w, const int* mel_lo, const int* mel_hi, int frame_len,
            int frame_shift, int log2_nfft, int snip_edges, int remove_dc, float preemph, float* feats, float dither,
            unsigned int dither_seed, void* stream, const float* dct, int num_ceps, int use_energy, int raw_energy,
            float energy_floor, int htk_compat);
int pk_frontend_fwd_mfcc(const short* pcm, long long ld_pcm, const int* n_samples, const float* rate, const int* new_len,
                         const float* target_db, const int* n_frames, int B, int n_max, int t_max, int n_mel, int lctx,
                         int rctx, int stride, const float* window, const float* twiddle, const float* mel_w,
                         const int* mel_lo, const int* mel_hi, int frame_len, int frame_shift, int log2_nfft, int snip_edges,
                         int remove_dc, float preemph, int cmn, const float* offset, const float* scale, int f0, int fs,
                         int t0, int ts, void* out, int out_dtype, short* wave_i16_out, void* workspace,
                         long long workspace_bytes, int* err_flag, float dither, unsigned int dither_seed, void* stream,
                         const short* noise, const int* noise_idx, const long long* noise_off, const double* snr,
                         const double* noise_rms_db, const short* rir, const long long* rir_off, const int* rir_len,
                         const int* rir_idx, int rir_max_len, const float* dct, int num_ceps, int use_energy,
                         int raw_energy, float energy_floor, int htk_compat);

/* scipy.signal.fftconvolve(x, h, "same") in float64 for ragged batches: x [B, ld_x] (lengths n_len), h [B, ld_h] (lengths
 * m_len, 1 <= m_len <= m_max <= 65536) -> y [B, ld_y], n_len[b] samples each (y may alias x).  Workspace:
 * pk_conv_same_f64_workspace_bytes (< 0 on bad dims). */
long long pk_conv_same_f64_workspace_bytes(int B, int n_max, int m_max);
int pk_conv_same_f64(const double* x, long long ld_x, const int* n_len, const double* h, long long ld_h, const int* m_len, int B,
                     int n_max, int m_max, double* y, long long ld_y, void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batched beam search (pika_b200/csrc/beam.cu): one launch per step for the whole batch.
 * Replaces decoder/beam_transducer.py:82-187 (BeamMergeTransducer.advance) and the gather / masked LSTM
 * update / state reordering of decoder/transducer_decoder.py:127-150,173-178,188-202.  Rows are
 * utterance-major (row = b*K + k); blank = blk, EOS = -1.
 * The loop is meant to be replayed from a CUDA graph, so nothing step-dependent is a kernel argument: step_ctx [2] int32 lives in
 * device memory -- step_ctx[0] = step index (the kernels address next_ys[step] / prev_ks[step] themselves), step_ctx[1] = 1 while
 * `not all(b.done() for b in beam)` (decoder/transducer_decoder.py:123) and the history buffers have room; pk_beam_step_end
 * advances / latches both at the end of a step and every kernel of a dead step is a no-op.  Initialise step_ctx = {0, 1}.
 */
int pk_beam_prepare(const int* next_ys, const int* step_ctx, int* t_idx, const void* enc, int dtype, int Tenc, int H, void* enc_hid,
                    const float* embed, int E, void* x_emb, int ld_x, int K, int blk, int rows, void* stream);
int pk_beam_lstm_cell(const float* gates, const int* next_ys, const int* step_ctx, int blk, void* h, int dtype, float* c, int rows, int H,
                      void* stream);
int pk_beam_step_end(int* step_ctx, const int* not_done, int max_steps, void* stream);
int pk_beam_gate(const float* a, void* h, int dtype, int rows, int H, void* stream);
/* one BeamMergeTransducer.advance for every utterance.  The word scores are given as the joint's logits [B*K rows, pitch ldv] f32 plus
 * the per-row log-sum-exp of sm_scale * logits (pk_row_lse): word_probs[r, v] = logits[r, v] * sm_scale - row_lse[r], the very expression
 * pk_log_softmax evaluates (decoder/transducer_decoder.py:177), formed on the fly so that the [B*K, V] log-prob tensor is never written.
 * t_idx [B*K], histories next_ys [S+1,B,K], prev_ks [S,B,K]; partial hypotheses hyp_tok [2,B,K,L] / hyp_len [2,B,K];
 * finished lists fin_* [B,cap]; *not_done_total is decremented when an utterance becomes done. */
int pk_row_lse(const void* x, int dtype, long long ld, float* lse, long long rows, int n, float scale, void* stream);
int pk_beam_advance(const float* logits, int ldv, const float* row_lse, float sm_scale, const int* t_idx, const int* num_frames, const int* max_len, float* scores,
                    int* next_ys, int* prev_ks, int* hyp_tok, int* hyp_len, float* fin_score, int* fin_step, int* fin_k,
                    int* fin_count, int* eos_top, int* done, int* not_done_total, int B, int K, int V, int L, int cap,
                    const int* step_ctx, int blk, int n_best, int beam_prune, void* stream);
int pk_beam_reorder(const int* prev_ks, const int* step_ctx, const void* h_in, const float* c_in, const int* t_in, void* h_out, float* c_out,
                    int* t_out, int dtype, int K, int H, int layers, int rows, void* stream);
/* On-the-fly FST shallow fusion inside the beam step: decoder/beam_transducer.py:135-159,167-176 with the arc search of
 * decoder/sorted_matcher.py:24-111 over a flattened arc table (arcs of a state sorted by input label, label = token + 1).
 * Per beam the active FST states are an insertion-ordered set of at most max_states (state, cost) pairs in double precision;
 * err_flag is raised when a set would overflow.  lm_scores [B,K] f32 and the sets ([2,B,K,max_states], [2,B,K]) are state the
 * caller zero-initialises before step 0. */
typedef struct {
    const int* arc_off;       /* [n_states + 1] */
    const int* arc_ilabel;    /* [n_arcs] */
    const double* arc_weight; /* [n_arcs] */
    const int* arc_next;      /* [n_arcs] */
    const double* finals;     /* [n_states], +inf = not final */
    int backoff_id, n_disambig;
    int disambig_ids[4];
} pk_lm_fst;
int pk_beam_advance_lm(const float* logits, int ldv, const float* row_lse, float sm_scale, const int* t_idx, const int* num_frames, const int* max_len, float* scores,
                       int* next_ys, int* prev_ks, int* hyp_tok, int* hyp_len, float* fin_score, int* fin_step, int* fin_k,
                       int* fin_count, int* eos_top, int* done, int* not_done_total, int B, int K, int V, int L, int cap,
                       const int* step_ctx, int blk, int n_best, int beam_prune, const pk_lm_fst* fst, double lm_scale, double nonblk_reward,
                       int* set_state, double* set_cost, int* set_n, float* lm_scores, int max_states, int* err_flag, void* stream);

/* Incremental step of the convolutional-transformer prediction net in the beam loop (pika_b200/csrc/beam_xf.cu): each row computes
 * only its newest position p against a KV cache, decoder/transducer_decoder.py:117-120,151-171 without re-running the history.
 * pool [n_entries][layers][3][D] (activation dtype): per layer the K row, the V row and (l >= 1) the layer's input, of one position;
 * entry 0 = the shared SOS position, entry 1 + s*rows + row = the position `row` computes at beam step s.  slot [2][rows][S1] int32:
 * position -> entry, ping-pong by step parity like hyp_tok [2][rows][S1] / hyp_len [2][rows].
 * A row computes in step s = step_ctx[0] when next_ys[s][row] > blk, at p = hyp_len[s&1][row]; other rows are masked at the writes.
 * init = 1: row 0 computes position 0 (token blk) into entry 0, and pk_beam_xf_select hands its output to every row. */
typedef struct {
    const int* next_ys;       /* [S+1][rows] */
    const int* step_ctx;      /* [2] */
    const int* hyp_tok;       /* [2][rows][S1] */
    const int* hyp_len;       /* [2][rows] */
    int* slot;                /* [2][rows][S1] */
    void* pool;               /* [n_entries][layers][3][D] */
    long long n_entries;
    int blk, rows, S1, layers, D, dtype, init;
} pk_beam_xf_state;
/* taps [rows][5*ldc]: the causal Conv1d(k=5) im2col row of position p (x(p-4) .. x(p), zero before position 0).  Layer 0: embedding rows
 * (f32 table [*, E]) of the tokens; layer >= 1: x_cur [rows][D] at p (also stored into the row's pool entry), the pool before it. */
int pk_beam_xf_taps(const pk_beam_xf_state* st, int layer, const float* embed, int E, const void* x_cur, void* taps, int ldc, void* stream);
/* qkv [rows][3D] (q | k | v) -> out [rows][D]: stores K / V of position p, attends over positions 0..p (fp32 online softmax, scale 1/8);
 * head size 64 only.  max_rel > 0: relative positions, rel f32 [2*max_rel+1][64] shared by keys and values. */
int pk_beam_xf_attn(const pk_beam_xf_state* st, int layer, const void* qkv, int heads, const float* rel, int max_rel, void* out, void* stream);
/* h[row] = x[row] [rows][H] on the rows that computed a position */
int pk_beam_xf_select(const pk_beam_xf_state* st, const void* x, void* h, int H, void* stream);
/* after pk_beam_advance[_lm] of step s: slot[s&1^1][row] = slot[s&1][src] up to src's length (src = prev_ks[s][row], or row if it finished) */
int pk_beam_xf_slots(const pk_beam_xf_state* st, const int* prev_ks, int K, void* stream);

/* ------------------------------------------------------------------------------------------
 * Persistent LSTM layer (pika_b200/csrc/lstm_seq.cu): the whole recurrence of one nn.LSTM layer in one
 * cooperative launch per 32 sequences (trainer/model/transducer.py:56-61,95), zero initial state.
 *   fwd: gx f32 [B,U,4H] = x W_ih^T + b_ih + b_hh; w_hh bf16 [4H,H]; out [B,U,H] (f32|bf16);
 *        gates_save f32 [U,B,4H], cs f32 [U,B,H] are kept for the backward.
 *   bwd: dout [B,U,H] -> dG bf16 [U,B,4H] (gradient w.r.t. the pre-activation gates, time-major).
 *   ws : pk_lstm_seq_workspace_bytes(H) bytes of zero-initialised scratch (grid barrier + hidden-state exchange).
 */
long long pk_lstm_seq_workspace_bytes(int H);
/* Ragged, (bi)directional form (the LSTM encoder over pack_padded_sequence batches; trainer/model/transducer.py:38-44,82-86).
 * n_dir = 2 runs both directions of a bidirectional layer in one launch of 2 * H/8 CTAs; n_dir = 1 with reverse = 1 runs one
 * direction backwards in time.  Per direction d (buffers stacked along a leading n_dir axis): gx f32 [B,U,4H], w_hh bf16 [4H,H],
 * gates_save f32 [U,B,4H], cs f32 [U,B,H], dG bf16 [U,B,4H]; out / dout [B,U,ldo], direction d at columns [d*H, (d+1)*H).
 * lens: int32 [B] on the device, or NULL (every sequence runs all U steps).  Sequence b with length L_b is processed at
 * t = s (forward) or t = L_b - 1 - s (reverse) for steps s < L_b, from a zero state; the kernel runs max_b L_b steps.
 * Outputs and dG rows at t >= L_b are written as zeros.  ws: pk_lstm_seq_workspace_bytes(n_dir * H) bytes, zero-initialised.
 * w_hh (fwd), dG (bwd) and ws must be 16-byte aligned; H a multiple of 64 with n_dir * H/8 <= #SMs; B, U >= 1; ldo >= n_dir * H.
 * The prediction net's layer is the lens = NULL, n_dir = 1, reverse = 0, ldo = H case. */
int pk_lstm_seq_fwd_ex(const float* gx, const void* w_hh_bf16, void* out, int out_dtype, int ldo, float* gates_save, float* cs,
                       const int* lens, int B, int U, int H, int n_dir, int reverse, void* ws, void* stream);
int pk_lstm_seq_bwd_ex(const void* dout, int dtype, int ldo, const float* gates_save, const float* cs, const void* w_hh_bf16,
                       void* dG_bf16, const int* lens, int B, int U, int H, int n_dir, int reverse, void* ws, void* stream);

/* ------------------------------------------------------------------------------------------
 * MBR training step helpers (trainer/train_transducer_mbr_bmuf_otfaug.py:197-235): the joint is evaluated only
 * on the (t,u) nodes of each N-best alignment, so rows are gathered, and the sparse mbr_grad through
 * log_softmax(sm_scale * out) is formed directly.
 */
int pk_gather_rows(const void* src, const int* idx, void* dst, int dtype, long long rows, int C, void* stream);
int pk_scatter_add_rows(const void* src, const int* idx, float* dst, int dtype, long long rows, int C, void* stream);
/* dz[r] = scale * coef[r] * (onehot(tok[r]) - softmax(scale * z[r]));  z, dz [rows, ld], first n columns valid */
int pk_ce_grad(const void* z, int dtype, long long ld, const int* tok, const float* coef, float scale, void* dz,
               long long rows, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
