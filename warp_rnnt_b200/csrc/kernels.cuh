// kernels.cuh -- host-side launch entry points shared between the .cu files and api.cu.
#pragma once
#include "common.cuh"

namespace rnnt {

void count_launch();   // api.cu: bumps the library-wide launch counter
// api.cu: test hook (rnnt_b200_debug_guard_poison): sample index whose alpha-side log-likelihood gets `delta` added
// in front of the forward/backward mismatch guard; n < 0 = off
struct GuardPoison { int n; float delta; };
GuardPoison guard_poison();
// api.cu: the calling thread's record of its last recurrence launch (rnnt_b200_debug_last_launch), indexed by
// rnntLaunchRecord_t.  begin_launch_record(path) clears it, counts the launch and sets the path (1 fused, 2 general).
int32_t *launch_record();
void begin_launch_record(int path);

cudaError_t launch_prefix(cudaStream_t s, const int *xn, const int *yn, int N, int64_t *mem_pref,
                          int64_t *lab_pref, int *totals);
// Compact grids are (gx, N): lattice lengths are on the device only, so gx covers twice the average lattice
// (STU / N rows, as launch_gather sizes its grid) in CTAs of kCompactIters grid-stride iterations each; a larger lattice
// is finished by the grid stride, the surplus CTAs of a smaller one return at once.
constexpr int64_t kCompactIters = 4;
inline int compact_gx(int64_t STU, int N, int64_t per_cta_rows) {
    const int64_t per = (STU / (N > 0 ? N : 1)) * 2 + 1;
    return (int)max((int64_t)1, min((per + per_cta_rows - 1) / per_cta_rows, (int64_t)65535));
}
// The LSE flavour of a launch: the fast one, else the reference's exact formula of the layout (dense or compact).
inline int lse_kind(bool fast_lse, bool compact) { return fast_lse ? kFast : compact ? kExactCompact : kExactDense; }

cudaError_t launch_gather(cudaStream_t s, const Problem &p, const void *lp, const int *labels, int V, int blank,
                          float2 *pairs, int64_t *loc, int64_t cells_hint, int io_bf16);
// the LSE kind follows p's layout; the forward/backward mismatch guard runs on the dense layout only (the compact
// reference has none, core_compact.cu:347-358)
cudaError_t launch_wavefront(cudaStream_t s, bool fast_lse, const Problem &p, const float2 *pairs, float *alphas,
                             float *betas, float *ws_ll, int *bad, float *costs, int beta_only, int t_hint,
                             int u_hint);
// Viterbi alignment (k_align): pairs -> alpha (workspace), decision words dec (N, ceil(U/32), T+31), scores (N) and
// frames (dense (N,U-1), compact (sum yn)); T, U bound the lattices (compact: max_T, max_U > 0)
cudaError_t launch_align(cudaStream_t s, const Problem &p, const float2 *pairs, float *alphas, uint32_t *dec, int T,
                         int U, float *scores, int *frames);
cudaError_t launch_grads_pairs(cudaStream_t s, const Problem &p, const float2 *pairs, const float *alphas,
                               const float *betas, const int *bad, float fastemit_lambda, float2 *out,
                               int64_t cells_hint);

// expand.cu -- dense gradient emit (every element of `out` is written)
struct ExpandSrc {
    // source A: alpha/beta/pairs (forward, dense layout)      -> pg == nullptr
    // source B: pair grads (cells,2) (+ per-sample scale)     -> pg != nullptr
    const float2 *pairs;
    const float *alphas;
    const float *betas;
    const int *bad;
    const float2 *pg;
    const float *scale;      // (N) or nullptr
    const int *labels;       // dense: (N,U-1)
    const int64_t *loc;      // compact backward: label id per cell (blank on the last column)
    const int *cum_lens;     // compact backward: inclusive cumsum of xn*(yn+1), (N)
    float fastemit_lambda;
    int label_adds;          // 1: label == blank accumulates (torch scatter_add semantics of gather=True)
};
cudaError_t launch_expand(cudaStream_t s, const Problem &p, const ExpandSrc &src, void *out, int64_t cells,
                          int V, int blank, bool retire_early, int io_bf16);   // io_bf16: bf16 output (forward emit)

// logits.cu -- loss from un-normalised logits (fused log_softmax forward / backward).  io_bf16: the logits (and the
// gradient written by launch_expand_logits) are bf16, else float; lse, pairs, pg and grad_out are float either way.
// hat: the HAT normalisation (logits.cu) in the k_*_hat kernels instead of log_softmax.
cudaError_t launch_lse_pairs(cudaStream_t s, const void *x, const int *labels, int N, int T, int U, int V, int blank,
                             float2 *pairs, float *lse, int io_bf16, int hat);
cudaError_t launch_expand_logits(cudaStream_t s, const void *x, const float *lse, const float2 *pg, const int *labels,
                                 const float *grad_out, void *out, int N, int T, int U, int V, int blank,
                                 int io_bf16, int hat);
// ... the same two passes over compact (STU,V) logits in joint_pack's row order: p is the compact Problem (prefix sums
// on the device), labels (sum yn), grad_out (N) or nullptr
cudaError_t launch_lse_pairs_compact(cudaStream_t s, const void *x, const Problem &p, const int *labels, int64_t STU,
                                     int V, int blank, float2 *pairs, float *lse, int io_bf16, int hat);
cudaError_t launch_expand_logits_compact(cudaStream_t s, const void *x, const float *lse, const float2 *pg,
                                         const Problem &p, const int *labels, const float *grad_out, void *out,
                                         int64_t STU, int V, int blank, int io_bf16, int hat);
// ... and over rnnt_loss_pruned's (N,T,S,V) window rows: row (n,t,s) is cell (t, ranges[n,t] + s) of the full (N,T,U)
// lattice.  The forward writes lse (N,T,S) and the full (N,T,U,2) pairs: every cell (kBig, kBig), then each window
// row's pair at its cell (u in [0, U)); the backward writes (N,T,S,V) from the full (N,T,U,2) pair gradients.
cudaError_t launch_lse_pairs_pruned(cudaStream_t s, const void *x, const int *labels, const int *ranges, int N, int T,
                                    int S, int U, int V, int blank, float2 *pairs, float *lse, int io_bf16, int hat);
cudaError_t launch_expand_logits_pruned(cudaStream_t s, const void *x, const float *lse, const float2 *pg,
                                        const int *labels, const int *ranges, const float *grad_out, void *out, int N,
                                        int T, int S, int U, int V, int blank, int io_bf16, int hat);

// simple.cu -- the simple (factorised-joint) loss: am (N,T,V) + lm (N,U,V), and the prune ranges of its lattice
struct SimpleArgs {
    const float *am, *lm;              // (N,T,V), (N,U,V)
    const int *labels, *xn, *yn;       // (N,U-1), (N), (N)
    float *norm, *off_a, *off_l;       // (N,T,U), (N,T), (N,U): written by the forward, read by the backward
    float2 *pairs;                     // forward: (N,T,U) (blank, label) log-probs out
    const float2 *pg;                  // backward: (N,T,U) pair gradients
    const float *grad_out;             // backward: (N), or null (ones)
    float *out;                        // the contraction's output (set by launch_simple_backward)
    int T, U, V, blank;
};
// row offsets, Z and the epilogue: norm and the pairs of every cell (0 outside the lattice)
cudaError_t launch_simple_forward(cudaStream_t s, const SimpleArgs &a, int N);
// dam (N,T,V) and dlm (N,U,V), every element written
cudaError_t launch_simple_backward(cudaStream_t s, const SimpleArgs &a, float *dam, float *dlm, int N);
// k2's smoothed simple loss (lm_only_scale sl, am_only_scale sa, c = 1 - sl - sa): the extra row passes, the batch
// unigram and the mixed pairs (forward), and the sl / sa / unigram gradient terms (backward)
constexpr int kSmoothRows = 32;        // rows per CTA of the unigram and G partials: the partition depends on shapes only
struct SmoothArgs {
    const float *am, *lm;              // (N,T,V), (N,U,V)
    const int *labels, *xn, *yn;       // (N,U-1), (N), (N)
    const float *off_a, *off_l;        // oa (N,T), ol (N,U) of the simple forward
    float *Ll, *Am, *loguni;           // saved: (N,U), (N,T), (V)
    float *uni, *upart;                // forward workspace: uni (V), unigram partials (ceil(N*U / kSmoothRows), V)
    float2 *pairs;                     // forward: the simple pairs in, the mixed pairs out
    const float2 *pg;                  // backward: (N,T,U) pair gradients
    const float *grad_out;             // backward: (N), or null (ones)
    float *cgo, *cb, *cl, *gpart, *G;  // backward workspace: c*grad_out (N), column sums of gb, gl (N,U), G partials
                                       // (ceil(N*T / kSmoothRows), V), G (V)
    float c, sl, sa;
    int N, T, U, V, blank;
};
// after launch_simple_forward: Ll (and, with sa > 0, uni, log uni, Am), then the mixed pairs in place
cudaError_t launch_simple_smoothed_forward(cudaStream_t s, const SmoothArgs &m);
// column sums and c*grad_out; launch_simple_backward on c*grad_out; then the sa (am rows, G) and sl / unigram (lm rows)
// terms added to dam, dlm
cudaError_t launch_simple_smoothed_backward(cudaStream_t s, const SimpleArgs &a, const SmoothArgs &m, float *dam,
                                            float *dlm);
// ranges (N,T) from the pair gradients (N,T,U,2) of a loss call; rnnt_type 0 (S >= 2), 1 or 2 (S >= 1); raw_blank:
// the constrained call's blank slots before the fold (N,T,U), read for rnnt_type 2 only
cudaError_t launch_prune_ranges(cudaStream_t s, const float2 *pg, const float *raw_blank, const int *xn, const int *yn,
                                int N, int T, int U, int S, int rnnt_type, int *ranges);

// frames.cu -- k2's modified / constrained lattices and delay penalty on the dense (N,T,U,2) pairs
constexpr int kFramesMaxU = 25600;        // k_frames keeps two rows of U floats in shared memory
struct FramesCall {
    const float2 *pairs;                  // (N,T,U,2) (blank, label) log-probs
    const int *xn, *yn;
    float *alphas, *betas, *ll;           // workspace: (N,T,U), (N,T,U), (N)
    int *status;                          // workspace: (N) lattice class
    float *costs;
    float2 *pair_grads;                   // (N,T,U,2) out, or null (costs only)
    float *raw_blank;                     // (N,T,U) out: blank slots before the constrained fold, or null
    int N, T, U;
    bool constrained;
};
// pairs_out = pairs_in with lam * ((Tn-1)/2 - t) added to every live label slot (in place when they are the same)
cudaError_t launch_delay_pairs(cudaStream_t s, const float2 *pairs_in, float2 *pairs_out, const int *xn, const int *yn,
                               int N, int T, int U, float lam);
// k_frames then, with pair_grads, k_frames_grads; `delayed` is recorded (the call ran launch_delay_pairs first)
cudaError_t launch_frames(cudaStream_t s, const FramesCall &c, bool delayed);
void frames_launch_record(int32_t *out);  // copy of the last k_frames launch's record (rnntFramesLaunchRecord_t)
// Viterbi alignment on the modified / constrained lattice (k_frames_align): pairs -> decision words dec
// (N, ceil(U/32), T), scores (N) and frames (N, U-1)
struct FramesAlignCall {
    const float2 *pairs;                  // (N,T,U,2) (blank, label) log-probs, penalised already when `delayed`
    const int *xn, *yn;
    uint32_t *dec;                        // workspace: frames_align_words(N, T, U) words
    float *scores;
    int *frames;
    int N, T, U;
    bool constrained, delayed;            // `delayed` is only recorded
};
inline size_t frames_align_words(int N, int T, int U) {
    return (size_t)max(N, 0) * (size_t)((max(U, 0) + 31) / 32) * (size_t)max(T, 0);
}
cudaError_t launch_frames_align(cudaStream_t s, const FramesAlignCall &c);
void frames_align_launch_record(int32_t *out);   // copy of the last k_frames_align launch's record

// joint.cu -- compact packing of the joint network's input (caller side of compact=True)
cudaError_t launch_joint_pack(cudaStream_t s, const float *f, const float *g, const int *lf, const int *lg,
                              const int64_t *mem_pref, float *x, int N, int T, int U1, int H, int64_t stu_hint);
cudaError_t launch_joint_grads(cudaStream_t s, const float *dx, const int *lf, const int *lg, const int64_t *mem_pref,
                               float *df, float *dg, int N, int T, int U1, int H);

// fused.cu -- single-kernel path for lattices that fit shared memory
// Wd: staged row stride (floats); nd: staged diagonals; C: lattice columns per lane (1, 2 or 4); slices: CTAs per
// lattice; smem: dynamic shared memory of the staged lattice and the zero buffer (bytes; launch_fused adds the TMA
// row buffers)
struct FusedPlan { int Wd, nd, C, slices; size_t smem; };
bool fused_plan(int N, int T, int U, FusedPlan *plan);
void set_fused_trace(long long *buf);   // diagnostics: per-CTA phase stamps of k_fused (8 x clock64 per CTA)
// One fused launch, filled by name; fields left zero are off.  The layout follows mem_pref: null = dense (N,T,U),
// with the mismatch guard; set = compact (T, U = max lengths), without it.  The LSE kind follows fast_lse and the layout.
struct FusedCall {
    bool fast_lse;
    const void *lp;                       // log-probs (N,T,U,V) or compact (STU,V); pairs_in: (cells,2) f32 pairs
    const int *labels;                    // dense (N,U-1), compact (sum yn); null with pairs_in
    const int *xn, *yn;
    const int64_t *mem_pref, *lab_pref;   // compact: first cell / first label of lattice n
    int64_t *loc;                         // compact: label id per cell, or null
    float *costs;
    void *grads;                          // dense gradient (N,T,U,V) of the element type, or null
    float2 *pair_grads;                   // (cells,2) gradient, or null
    const float *scale;                   // (N) or null
    float *loss_sum;                      // sum_n costs[n]*scale[n] in the kernel; needs sync_counter
    unsigned *sync_counter;
    int N, T, U, V, blank;
    float lam;
    int pairs_in;
    int io_bf16;                          // log_probs and the dense gradient are bf16 (dense gradient only)
};
cudaError_t launch_fused(cudaStream_t s, const FusedPlan &plan, const FusedCall &c);

// tdt.cu -- the Token-and-Duration Transducer loss from (N,T,U,V+D) joint logits, and on the same kernels the
// multi-blank transducer loss from (N,T,U,V) logits (include/rnnt_b200.h)
constexpr int kTdtMaxD = 17;              // durations are distinct values in [0, 16]
struct TdtDurations { int d[kTdtMaxD]; int D, dmax; };
// the launch shape the planner picks (recorded by rnnt_b200_debug_last_tdt_launch)
struct TdtPlan {
    int norm_group, norm_lanes;           // normaliser: elements per load (4, 2, 1), lanes per row (8, 32)
    int kd;                               // recurrence / posterior instantiation: candidate slots (5 or kTdtMaxD)
    int warps, passes;                    // recurrence: warps per CTA, column passes per diagonal
    int ring, smem;                       // ring slots in shared memory (0: read back from global), its bytes
};
// multiblank: dur holds the big blanks' durations and V is the whole row
TdtPlan tdt_plan(int U, const TdtDurations &dur, const void *x, int elem_bytes, int V, bool multiblank = false);
// The compact layout of a TDT call (joint_pack's row order): lattice n is a Tn x Un slab at row mem_pref[n] with row
// stride Un = yn[n] + 1, its labels start at lab_pref[n]; a lattice is ok when Tn <= max_T, Un <= max_U and its rows lie
// inside [0, STU).  The backward takes max_T = max_U = 0 (it does not check lattices: the posteriors tell).
struct TdtCompact {
    const int64_t *mem_pref, *lab_pref;
    int64_t STU;
    int N, max_T, max_U;
};
// Every field below that names a (N,T,U,...) shape is (STU,...) in the compact layout (mem_pref set), where T and U are
// the bounds max_T, max_U and labels is (sum yn).  multiblank: the multi-blank lattice, with dur the big blanks'
// durations (D = B), V the whole row (blank in [B, V)), lse_mb (N,T,U) out in place of lse, and pg (N,T,U,2+B) =
// (P_std, Pl, P_big[0..B)).
struct TdtFwd {
    const void *x;                        // logits (N,T,U,V+D), f32 or bf16
    const int *labels, *xn, *yn;
    const int64_t *mem_pref, *lab_pref;   // compact: the prefix sums of xn * (yn + 1) and yn; null: dense
    int64_t STU;                          // compact: rows
    float *costs;
    float2 *lse;                          // (N,T,U) (lse_tok, lse_dur) out
    float *pg;                            // (N,T,U,2+D) posteriors out, or null (costs only)
    float *lp, *alpha, *beta, *ll;        // workspace: (N,T,U,2+D), (N,T,U), (N,T,U), (N)
    int *status;                          // workspace: (N) lattice class
    int N, T, U, V, blank;
    float sigma;
    TdtDurations dur;
    int io_bf16;
    bool multiblank;
    float *lse_mb;                        // multiblank: (N,T,U) lse out
};
cudaError_t launch_tdt_forward(cudaStream_t s, const TdtFwd &c);
struct TdtBwd {
    const void *x;                        // logits (N,T,U,V+D)
    const float2 *lse;
    const float *pg;                      // (N,T,U,2+D) posteriors of the forward
    const int *labels;
    const int *yn;                        // compact only, with mem_pref, lab_pref and STU as in TdtFwd
    const int64_t *mem_pref, *lab_pref;
    int64_t STU;
    const float *grad_out;                // (N), or null (ones)
    void *out;                            // (N,T,U,V+D), of the logits' type
    int N, T, U, V, D, blank;
    int io_bf16;
    bool multiblank;                      // as in TdtFwd: V the whole row, D = B
    const float *lse_mb;                  // multiblank: (N,T,U) lse of the forward
};
cudaError_t launch_tdt_backward(cudaStream_t s, const TdtBwd &c);
// The Viterbi alignment on the TDT lattice (rnnt_b200_tdt_align_*): c as for the forward, with costs = the scores
// (N) and pg, beta, ll unused; the normaliser writes lse and lp, then k_tdt_align writes alpha, dec (cells bytes, the
// decision per cell), status, the scores, and frames and fdur (dense (N,U-1), compact (sum yn)).
cudaError_t launch_tdt_align(cudaStream_t s, const TdtFwd &c, uint8_t *dec, int *frames, int *fdur);
// The Viterbi alignment on the multi-blank lattice (rnnt_b200_multiblank_align_*): c as for the multiblank forward
// (lse_mb the normaliser's (cells) floats), costs = the scores (N), pg, beta, ll unused; k_mb_align writes alpha, dec,
// status, the scores, frames (dense (N,U-1), compact (sum yn)) and counts (N, 1 + B).
cudaError_t launch_mb_align(cudaStream_t s, const TdtFwd &c, uint8_t *dec, int *frames, int *counts);
void tdt_launch_record(int32_t *out);     // copy of the last TDT launch's record (rnntTdtLaunchRecord_t)

// expand.cu -- small helpers of the python-level API
cudaError_t launch_loss_sum(cudaStream_t s, const float *costs, const float *scale, int N, float *loss_sum);
cudaError_t launch_rescale(cudaStream_t s, void *grads, const float *grad_out, int grad_out_stride,
                           const float *applied, int N, int64_t elems_per_sample, int io_bf16);

}  // namespace rnnt
