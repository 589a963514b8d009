// tdt.cu -- the Token-and-Duration Transducer loss (TDT, Xu et al. 2023, arXiv:2304.06795) from joint logits.
//
// A TDT joint gives, per lattice cell, V token logits and D duration logits (NeMo's layout: row width W = V + D).  A
// token emitted with duration d moves the path d frames ahead, so the recurrence looks back up to max(d) frames.  The
// semantics (edges, classes of degenerate input) are stated in include/rnnt_b200.h.  Three stages, as the from-logits
// path of logits.cu:
//
//   k_tdt_norm   one read of every live row: two online max / sum reductions (tokens, durations) -> lse (N,T,U,2) and
//                the 2 + D f32 log-probs the recurrence needs, lp (N,T,U,2+D) = (blank - sigma, label - sigma, ld[0..D)),
//                each clamped below at kBig (a masked -inf becomes the finite sentinel)
//   k_tdt_recur  one CTA per lattice and direction (grid (N, 2)): alpha (blockIdx.y = 0) and beta (1) along
//                anti-diagonals s = t + u, threads over columns; the last max(d) + 2 diagonals in a shared-memory ring
//                (or, when the ring does not fit, read back from the alpha / beta arrays in global memory).  The beta
//                CTA also classifies the lattice and writes its cost.
//   k_tdt_post   per cell, the edge posteriors -> (Pb, Pl, Pd[0..D)) (N,T,U,2+D), unscaled
//   k_tdt_emit   (backward) one read of the logits and one write of d loss / d logits (N,T,U,V+D), every element once
//   k_tdt_align  (rnnt_b200_tdt_align_*, after k_tdt_norm) the Viterbi alignment: one CTA per lattice (grid (N, 1)),
//                tdt_recur's alpha side in max-plus form with a decision byte per cell, then the class, the score and
//                the backtrace in the same kernel
//
// Every LSE is one max-then-sum over all candidate terms of a cell.  All candidates are finite (kBig sentinels) or NaN,
// absent ones are -inf and only ever subtracted from a finite maximum: -inf - -inf is never formed.  No atomics: every
// value has one writer and a fixed operation order, so results are deterministic.  A bf16 row is read in exactly the
// f32 row's order (branch and lanes depend on the row width and the element alignment only), so lse, lp, costs and the
// posteriors are bit for bit those of the widened logits, and the bf16 gradient is the f32 gradient rounded once.
//
// Compact layout (joint_pack's row order, rnnt_b200_tdt_compact_*): the logits are (STU, V+D) and every intermediate
// is compact too -- lse (STU,2), lp and the posteriors (STU,2+D), alpha / beta (STU).  Lattice n is a Tn x Un slab at
// row mem_pref[n] with row stride Un, its labels start at lab_pref[n]; T and U are the bounds max_T, max_U.  Each
// kernel body is shared by the two layouts and takes the layout as a template flag (COMPACT): only the cell ->
// (n, t, u) mapping differs, so a compact row is computed exactly as the same row of a padded tensor.  The normaliser
// runs one lattice per blockIdx.y (as logits.cu's compact rows); the posterior pass and the emit stay flat over the rows
// and find a row's lattice by a binary search of mem_pref (tdt_find).
//
// Multi-blank transducer (Xu et al. 2022, arXiv:2211.03541; rnnt_b200_multiblank_*): the same four stages on the same
// bodies, under the template flag MB, with B big blanks of durations d[0..B) in the durations' place (D = B).  The row
// is V logits with one normaliser (W = V), lse is (cells) floats and lp, the posteriors (cells, 2 + B) = (standard
// blank, label, big blank [0..B)), big blank i at column blank - 1 - i.  The edges out of (t, u): the standard blank to
// (t + 1, u), the label to (t, u + 1) and big blank i to (t + d[i], u), so alpha's sources lie on diagonals s - 1 and
// s - d[i] and the ring keeps max(d) + 1 diagonals.  Kernels k_mb_norm, k_mb_recur, k_mb_post, k_mb_emit (and their
// _compact twins); every TDT instantiation is the code it was.  k_mb_align (rnnt_b200_multiblank_align_*, after
// k_mb_norm) is the Viterbi alignment on this lattice: k_mb_recur's alpha side in max-plus form, as k_tdt_align is
// k_tdt_recur's, with the blank counts of the best path beside its label frames.
#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kTdtRowThreads = 256;   // k_tdt_norm, k_tdt_post, k_tdt_emit
constexpr int kTdtMaxThreads = 512;   // k_tdt_recur: at most 16 warps over the columns, then column passes

// lattice classes, written by the beta CTA (status (N) in the workspace)
enum { kTdtOk = 0, kTdtInvalid = 1, kTdtNan = 2, kTdtDead = 3 };

__device__ __forceinline__ float clamp_big(float v) { return v < kBig ? kBig : v; }   // NaN stays NaN

// lattice n of a compact call: ok when its lengths are in [1, max_T] x [1, max_U] and its rows lie inside [0, STU)
__device__ __forceinline__ Lattice tdt_lattice(const int *xn, const int *yn, const TdtCompact &cp, int n) {
    Lattice L;
    L.Tn = xn[n];
    L.Un = yn[n] + 1;
    L.stride = L.Un;
    L.base = cp.mem_pref[n];
    L.lab_base = cp.lab_pref[n];
    L.ok = L.Tn >= 1 && L.Tn <= cp.max_T && L.Un >= 1 && L.Un <= cp.max_U && L.base >= 0 &&
           L.base + (int64_t)L.Tn * L.Un <= cp.STU;
    return L;
}
// the compact lattice holding row r: the last n with mem_pref[n] <= r (the prefix sums do not decrease, so an empty
// lattice shares its first row with the next one and is passed over), -1 if there is none.  The caller still checks
// that r lies inside it.
__device__ __forceinline__ int tdt_find(const int64_t *__restrict__ mem_pref, int N, int64_t r) {
    int lo = 0, hi = N;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(mem_pref + mid) <= r) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// online max / sum: the running max m stays -inf while every element seen is -inf; until a finite one arrives the
// sum subtracts 0 instead (exp(-inf) = 0), so -inf - -inf is never formed.  A NaN makes the sum NaN, +inf too.
__device__ __forceinline__ void online_add(float &m, float &s, float a) {
    if (a > m) { s = s * expf(m - a); m = a; }
    s += expf(a - (m == -INFINITY ? 0.0f : m));
}
__device__ __forceinline__ void online_merge(float &m, float &s, float m2, float s2) {
    const float mm = fmaxf(m, m2);
    s = (m == mm ? s : s * expf(m - mm)) + (m2 == mm ? s2 : s2 * expf(m2 - mm));
    m = mm;
}
// every element -inf: NaN, as torch.log_softmax gives
__device__ __forceinline__ float online_lse(float m, float s) { return m == -INFINITY ? NAN : m + logf(s); }

// Normaliser pass.  SUB lanes per row (8 or 32), groups of G elements per load (4: rows of whole groups at group-aligned
// addresses, 2: the same for pairs, 1: any row); lanes stride over the groups, each lane keeps a token and a duration
// accumulator (an element goes to the one of its column), then a butterfly merges the lanes.  Lane 0 writes lse and lp.
// Rows outside the live lattice (padding, or a lattice with invalid lengths) are not read: lse (0, 0), lp untouched.
// COMPACT: CTA row blockIdx.y streams over the Tn * Un rows of lattice n, the pointers rebased to its first row; the rows
// of a lattice that is not ok are not read and lse / lp are not written there (the posteriors of those rows are 0).
// MB (LSE = float): one accumulator over the whole row of V; lp = (blank, label, big blanks) each minus sigma.
template <typename IN, int SUB, int G, bool COMPACT, bool MB = false, typename LSE = float2>
__device__ __forceinline__ void
tdt_norm_rows(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ xn,
              const int *__restrict__ yn, int64_t cells, int T, int U, int V, int D, int blank, float sigma,
              FastDiv divU, FastDiv divTU, LSE *__restrict__ lse, float *__restrict__ lp, const TdtCompact &cp) {
    const int W = MB ? V : V + D, W2 = 2 + D;
    Lattice L;
    if constexpr (COMPACT) {
        L = tdt_lattice(xn, yn, cp, blockIdx.y);
        cells = L.ok ? (int64_t)L.Tn * L.Un : 0;
        x += L.base * W; lse += L.base; lp += L.base * W2; labels += L.lab_base;
    }
    const int sub = threadIdx.x % SUB;
    const int64_t per_block = kTdtRowThreads / SUB;
    for (int64_t base = (int64_t)blockIdx.x * per_block; base < cells; base += (int64_t)gridDim.x * per_block) {
        const int64_t cell = min(base + threadIdx.x / SUB, cells - 1);   // surplus groups redo the last row
        uint32_t n, rem, t, u;
        int Tn, Un;
        bool live;
        if constexpr (COMPACT) {
            n = 0;                                                        // labels are rebased to the lattice's
            Tn = L.Tn; Un = L.Un;
            u = (uint32_t)cell % (uint32_t)Un;
            live = true;
        } else {
            divTU.divmod((uint32_t)cell, n, rem);
            divU.divmod(rem, t, u);
            Tn = xn[n]; Un = yn[n] + 1;
            live = Tn >= 1 && Tn <= T && Un >= 1 && Un <= U && (int)t < Tn && (int)u < Un;
        }
        const IN *row = x + cell * W;
        float mt = -INFINITY, st = 0.0f, md = -INFINITY, sd = 0.0f;
        if (live) {
            for (int q = sub; q < W / G; q += SUB) {
                float v[G];
                ld_logits<G>(row + q * G, v);
#pragma unroll
                for (int k = 0; k < G; ++k) {
                    if (MB || q * G + k < V) online_add(mt, st, v[k]);
                    else online_add(md, sd, v[k]);
                }
            }
        }
        if constexpr (MB) {
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) {
                const float mt2 = __shfl_xor_sync(0xffffffffu, mt, o), st2 = __shfl_xor_sync(0xffffffffu, st, o);
                online_merge(mt, st, mt2, st2);
            }
            if (sub != 0) continue;
            if (!live) {
                lse[cell] = 0.0f;
                continue;
            }
        } else {
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) {
                const float mt2 = __shfl_xor_sync(0xffffffffu, mt, o), st2 = __shfl_xor_sync(0xffffffffu, st, o);
                const float md2 = __shfl_xor_sync(0xffffffffu, md, o), sd2 = __shfl_xor_sync(0xffffffffu, sd, o);
                online_merge(mt, st, mt2, st2);
                online_merge(md, sd, md2, sd2);
            }
            if (sub != 0) continue;
            if (!live) {
                lse[cell] = make_float2(0.0f, 0.0f);
                continue;
            }
        }
        const float lt = online_lse(mt, st);
        float ld = 0.0f;
        if constexpr (MB) {
            lse[cell] = lt;
        } else {
            ld = online_lse(md, sd);
            lse[cell] = make_float2(lt, ld);
        }
        float *o = lp + cell * W2;
        o[0] = clamp_big((io_load(row + blank) - lt) - sigma);
        float l = kBig;                                         // the last column has no label edge
        if ((int)u < Un - 1) {
            const int lab = labels[(int64_t)n * (U - 1) + u];
            l = (lab >= 0 && lab < V) ? clamp_big((io_load(row + lab) - lt) - sigma) : NAN;   // bad label: k_tdt_recur
        }
        o[1] = l;
        if constexpr (MB) {
            for (int j = 0; j < D; ++j) o[2 + j] = clamp_big((io_load(row + blank - 1 - j) - lt) - sigma);
        } else {
            for (int j = 0; j < D; ++j) o[2 + j] = clamp_big(io_load(row + V + j) - ld);
        }
    }
}

template <typename IN, int SUB, int G>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_norm(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ xn,
           const int *__restrict__ yn, int64_t cells, int T, int U, int V, int D, int blank, float sigma, FastDiv divU,
           FastDiv divTU, float2 *__restrict__ lse, float *__restrict__ lp) {
    tdt_norm_rows<IN, SUB, G, false>(x, labels, xn, yn, cells, T, U, V, D, blank, sigma, divU, divTU, lse, lp,
                                     TdtCompact{});
}

// grid (gx, N): cells = STU
template <typename IN, int SUB, int G>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_norm_compact(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ xn,
                   const int *__restrict__ yn, int V, int D, int blank, float sigma, float2 *__restrict__ lse,
                   float *__restrict__ lp, TdtCompact cp) {
    tdt_norm_rows<IN, SUB, G, true>(x, labels, xn, yn, cp.STU, cp.max_T, cp.max_U, V, D, blank, sigma, FastDiv(),
                                    FastDiv(), lse, lp, cp);
}

// The multi-blank normaliser: lse (N,T,U), lp (N,T,U,2+B); D = B
template <typename IN, int SUB, int G>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_norm(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ xn,
          const int *__restrict__ yn, int64_t cells, int T, int U, int V, int D, int blank, float sigma, FastDiv divU,
          FastDiv divTU, float *__restrict__ lse, float *__restrict__ lp) {
    tdt_norm_rows<IN, SUB, G, false, true>(x, labels, xn, yn, cells, T, U, V, D, blank, sigma, divU, divTU, lse, lp,
                                           TdtCompact{});
}
template <typename IN, int SUB, int G>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_norm_compact(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ xn,
                  const int *__restrict__ yn, int V, int D, int blank, float sigma, float *__restrict__ lse,
                  float *__restrict__ lp, TdtCompact cp) {
    tdt_norm_rows<IN, SUB, G, true, true>(x, labels, xn, yn, cp.STU, cp.max_T, cp.max_U, V, D, blank, sigma,
                                          FastDiv(), FastDiv(), lse, lp, cp);
}

struct TdtRec {
    const float *lp;
    const int *labels, *xn, *yn;
    float *alpha, *beta, *ll, *costs;
    int *status;
    int T, U, V, D;
    int ring;                 // ring slots in shared memory (max(d) + 2, MB max(d) + 1), or 0: read back from alpha / beta
    TdtDurations dur;
};

// max-then-sum LSE over C candidates; absent ones are -inf.  No candidate: kBig (the cell has no edge).
template <int C>
__device__ __forceinline__ float lse_cands(const float (&c)[C]) {
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < C; ++k) m = fmaxf(m, c[k]);
    if (m == -INFINITY) return kBig;
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < C; ++k) s += expf(c[k] - m);          // a NaN candidate makes s NaN (fmaxf skipped it)
    return m + logf(s);
}

// The Viterbi alignment's outputs (k_tdt_align): the alpha side of tdt_recur in max-plus form.  Per cell, the index k
// in [0, 2 KD) of the candidate it took (2j: blank edge of duration d[j], 2j + 1: label edge), kTdtNoPred for (0, 0)
// and for a cell without a predecessor; frames / fdur: dense (N,U-1), compact (sum yn) in the labels' order.
constexpr int kTdtNoPred = 0xff;
struct TdtAlignOut {
    uint8_t *dec;                         // decisions, addressed as alpha
    int *frames, *fdur;
};
// The multi-blank alignment's outputs (k_mb_align): per cell the index k in [0, 2 + B) of the candidate it took (0:
// standard blank, 1: label, 2 + j: big blank j), kTdtNoPred as above; frames as above; counts (N, 1 + B): the standard
// blank's and each big blank's edges on the best path.
struct MbAlignOut {
    uint8_t *dec;
    int *frames, *counts;
};

// The largest of C candidates and its index in `arg`: blank edges (even k) first, then label edges (odd k), each by
// increasing duration, and only a strictly larger value replaces the one held, so on a tie blank beats label and the
// shorter duration wins.  Absent candidates are -inf and never taken.  No candidate: kBig and kTdtNoPred, as lse_cands.
// A NaN candidate is never taken either (the lattice is classed NaN whatever the sweep gives).
template <int C>
__device__ __forceinline__ float max_cands(const float (&c)[C], int &arg) {
    float m = -INFINITY;
    arg = kTdtNoPred;
#pragma unroll
    for (int k = 0; k < C; k += 2)
        if (c[k] > m) { m = c[k]; arg = k; }
#pragma unroll
    for (int k = 1; k < C; k += 2)
        if (c[k] > m) { m = c[k]; arg = k; }
    return arg == kTdtNoPred ? kBig : m;
}
// max_cands over the multi-blank layout (c[0] standard blank, c[1] label, c[2 + j] big blank j): the standard blank
// first, then the big blanks by increasing duration, then the label, so on a tie a blank beats the label and the
// shorter blank wins.  Absent and NaN candidates are never taken; no candidate: kBig and kTdtNoPred.
template <int C>
__device__ __forceinline__ float max_cands_mb(const float (&c)[C], int &arg) {
    float m = -INFINITY;
    arg = kTdtNoPred;
    if (c[0] > m) { m = c[0]; arg = 0; }
#pragma unroll
    for (int k = 2; k < C; ++k)
        if (c[k] > m) { m = c[k]; arg = k; }
    if (c[1] > m) { m = c[1]; arg = 1; }
    return arg == kTdtNoPred ? kBig : m;
}

// ALIGN, after the sweep, every thread of the CTA: the lattice's `slots` label slots at lab_base are set to -1; then,
// for a lattice classed ok, thread 0 follows the decisions back from the best terminal edge's source (t0, Un - 1) to
// (0, 0) and writes frame t and duration d of each label edge (t, u) -> (t + d, u + 1) into slot u.  A decision only
// ever names a predecessor that exists, so the walk stays inside the lattice; it is bounded by Tn + Un - 1 steps all
// the same (a path has at most Tn - 1 blank edges inside the lattice and Un - 1 label edges).
__device__ __forceinline__ void tdt_backtrace(const TdtRec &a, const TdtAlignOut &o, int64_t base, int ld,
                                              int64_t lab_base, int slots, int Tn, int Un, int t0, bool ok) {
    int *fr = o.frames + lab_base, *fd = o.fdur + lab_base;
    for (int u = threadIdx.x; u < slots; u += blockDim.x) {
        fr[u] = -1;
        fd[u] = -1;
    }
    __syncthreads();
    if (!ok || threadIdx.x != 0) return;
    int t = t0, u = Un - 1;
    for (int step = 0; step < Tn + Un - 1; ++step) {
        const int k = o.dec[base + (int64_t)t * ld + u];
        if (k == kTdtNoPred) break;
        const int d = a.dur.d[k >> 1];
        t -= d;
        if (k & 1) {
            --u;
            fr[u] = t;
            fd[u] = d;
        }
    }
}

// ALIGN && MB, after the sweep: as tdt_backtrace, the lattice's label slots set to -1 and, for a lattice classed ok,
// thread 0 follows the decisions back from the terminal edge k0 (0: the standard blank, 2 + j: big blank j) out of
// (t0, Un - 1) to (0, 0): k = 0 moves t back by 1, k = 1 moves u back by 1 and writes the label edge's frame, k = 2 + j
// moves t back by d[j].  The edge counts (terminal edge included) are kept in registers and written once to row n of
// o.counts; a lattice that is not ok gets -1 there.
template <int KD>
__device__ __forceinline__ void mb_backtrace(const TdtRec &a, const MbAlignOut &o, int64_t base, int ld,
                                             int64_t lab_base, int slots, int n, int Un, int t0, int k0, bool ok) {
    int *fr = o.frames + lab_base, *cnt = o.counts + (int64_t)n * (1 + a.D);
    for (int u = threadIdx.x; u < slots; u += blockDim.x) fr[u] = -1;
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (!ok) {
        for (int k = 0; k <= a.D; ++k) cnt[k] = -1;
        return;
    }
    int n_std = 0, n_big[KD - 2];
#pragma unroll
    for (int j = 0; j < KD - 2; ++j) n_big[j] = 0;
    int t = t0, u = Un - 1, k = k0;
    for (int step = 0; step <= t0 + Un - 1; ++step) {
        n_std += k == 0;
#pragma unroll
        for (int j = 0; j < KD - 2; ++j) n_big[j] += k == 2 + j;
        k = o.dec[base + (int64_t)t * ld + u];
        if (k == kTdtNoPred) break;
        if (k == 0) {
            --t;
        } else if (k == 1) {
            --u;
            fr[u] = t;
        } else {
            t -= a.dur.d[k - 2];
        }
    }
    cnt[0] = n_std;
#pragma unroll
    for (int j = 0; j < KD - 2; ++j)
        if (j < a.D) cnt[1 + j] = n_big[j];
}

// alpha (blockIdx.y == 0) or beta (1) of lattice blockIdx.x.  KD >= D: the candidate arrays' compile-time size.
// The ring holds U (dense: the padded width, compact: max_U) columns per diagonal; lp, alpha and beta are addressed
// with the lattice's row stride ld (dense U, compact Un).
// ALIGN (k_tdt_align, grid (N, 1)): the alpha side only, with max_cands in place of lse_cands and a decision byte per
// cell; it also checks every live cell's own lp row for NaN, as the beta side does.  After the sweep, the class and
// the score (a.costs) of the lattice, then the backtrace (tdt_backtrace).
// MB (k_mb_recur): the multi-blank edges; KD >= 2 + B is the candidate array's size (standard blank, label, big blanks).
// ALIGN && MB (k_mb_align, OUT = MbAlignOut): the same alpha side with max_cands_mb, the cell's own row checked for
// NaN, then the terminal step by max_cands_mb's tie rule and mb_backtrace.
template <int KD, bool COMPACT, bool ALIGN = false, bool MB = false, typename OUT = TdtAlignOut>
__device__ __forceinline__ void tdt_recur(const TdtRec &a, const TdtCompact &cp, const OUT &o = OUT{}) {
    extern __shared__ float ring[];
    const int n = blockIdx.x;
    const bool beta_side = !ALIGN && blockIdx.y == 1;
    int Tn, Un;
    bool ok;
    int64_t base, lab_base;
    if constexpr (COMPACT) {
        const Lattice L = tdt_lattice(a.xn, a.yn, cp, n);
        Tn = L.Tn; Un = L.Un; ok = L.ok; base = L.base; lab_base = L.lab_base;
    } else {
        Tn = a.xn[n]; Un = a.yn[n] + 1;
        ok = Tn >= 1 && Tn <= a.T && Un >= 1 && Un <= a.U;
        base = (int64_t)n * a.T * a.U; lab_base = (int64_t)n * (a.U - 1);
    }
    if (!ok) {
        if constexpr (ALIGN) {
            if (threadIdx.x == 0) {
                a.status[n] = kTdtInvalid;
                a.costs[n] = NAN;
            }
            // the label slots of lattice n: dense U - 1, compact yn[n] (none when it is negative)
            const int slots = COMPACT ? max(Un - 1, 0) : a.U - 1;
            if constexpr (MB) mb_backtrace<KD>(a, o, 0, 0, lab_base, slots, n, 0, 0, 0, false);
            else tdt_backtrace(a, o, 0, 0, lab_base, slots, 0, 0, 0, false);
        } else if (beta_side && threadIdx.x == 0) {
            a.status[n] = kTdtInvalid;
            a.costs[n] = NAN;
            a.ll[n] = NAN;
        }
        return;
    }
    const int U = a.U, W2 = 2 + a.D, D = a.D, R = a.ring;
    const int ld = COMPACT ? Un : U;
    const int *labels = a.labels + lab_base;
    float *out = (beta_side ? a.beta : a.alpha) + base;
    const float *lp = a.lp + base * W2;
    // the value of cell (t, u) on the diagonal whose ring slot is sl (computed on an earlier step)
    auto rd = [&](int t, int u, int sl) -> float { return R ? ring[sl * U + u] : out[(int64_t)t * ld + u]; };
    const int S = Tn + Un - 1;
    bool saw_nan = false;
    for (int step = 0; step < S; ++step) {
        const int s = beta_side ? S - 1 - step : step;
        const int slot = R ? s % R : 0;
        auto back = [&](int k) { const int q = slot - k; return q < 0 ? q + R : q; };
        auto fwd = [&](int k) { const int q = slot + k; return q >= R ? q - R : q; };
        for (int u = max(0, s - Tn + 1) + (int)threadIdx.x; u <= min(s, Un - 1); u += blockDim.x) {
            const int t = s - u;
            float c[MB ? KD : 2 * KD];
            float v;
            if constexpr (MB) {
                if (!beta_side) {
                    // pull: standard blank from (t-1, u) and label from (t, u-1), both on diagonal s-1; big blank j
                    // from (t-d[j], u) on s-d[j]; weights at the source cell
                    c[0] = c[1] = -INFINITY;
                    if (t > 0) c[0] = rd(t - 1, u, back(1)) + lp[((int64_t)(t - 1) * ld + u) * W2];
                    if (u > 0) c[1] = rd(t, u - 1, back(1)) + lp[((int64_t)t * ld + u - 1) * W2 + 1];
#pragma unroll
                    for (int j = 0; j < KD - 2; ++j) {
                        c[2 + j] = -INFINITY;
                        if (j < D) {
                            const int d = a.dur.d[j], tp = t - d;
                            if (tp >= 0) c[2 + j] = rd(tp, u, back(d)) + lp[((int64_t)tp * ld + u) * W2 + 2 + j];
                        }
                    }
                    if constexpr (ALIGN) {
                        // the cell's own row, for the NaN class (the beta side's check, here on the alpha side)
                        const float *r = lp + ((int64_t)t * ld + u) * W2;
                        saw_nan |= (r[0] != r[0]) || (u < Un - 1 && r[1] != r[1]);
#pragma unroll
                        for (int j = 0; j < KD - 2; ++j)
                            if (j < D) saw_nan |= r[2 + j] != r[2 + j];
                        int k = kTdtNoPred;
                        v = (t == 0 && u == 0) ? 0.0f : max_cands_mb(c, k);
                        o.dec[base + (int64_t)t * ld + u] = (uint8_t)k;
                    } else {
                        v = (t == 0 && u == 0) ? 0.0f : lse_cands(c);
                    }
                } else {
                    // push: the cell's own weights, beta of the destinations; a blank that reaches t = Tn from the
                    // last column is terminal (beta 0 after it)
                    const float *r = lp + ((int64_t)t * ld + u) * W2;
                    const float b = r[0], l = r[1];
                    const bool has_label = u < Un - 1;
                    saw_nan |= (b != b) || (has_label && l != l);
                    c[0] = t + 1 < Tn ? b + rd(t + 1, u, fwd(1)) : has_label ? -INFINITY : b;
                    c[1] = has_label ? l + rd(t, u + 1, fwd(1)) : -INFINITY;
#pragma unroll
                    for (int j = 0; j < KD - 2; ++j) {
                        c[2 + j] = -INFINITY;
                        if (j < D) {
                            const int d = a.dur.d[j], tq = t + d;
                            const float lb = r[2 + j];
                            saw_nan |= lb != lb;
                            if (tq < Tn) c[2 + j] = lb + rd(tq, u, fwd(d));
                            else if (tq == Tn && !has_label) c[2 + j] = lb;
                        }
                    }
                    v = lse_cands(c);
                }
            } else if (!beta_side) {
                // pull: blank from (t-d, u) for d > 0, label from (t-d, u-1) for every d; weights at the source cell
#pragma unroll
                for (int j = 0; j < KD; ++j) {
                    c[2 * j] = c[2 * j + 1] = -INFINITY;
                    if (j < D) {
                        const int d = a.dur.d[j], tp = t - d;
                        if (tp >= 0) {
                            if (d > 0) {
                                const float *r = lp + ((int64_t)tp * ld + u) * W2;
                                c[2 * j] = (rd(tp, u, back(d)) + r[0]) + r[2 + j];
                            }
                            if (u > 0) {
                                const float *r = lp + ((int64_t)tp * ld + u - 1) * W2;
                                c[2 * j + 1] = (rd(tp, u - 1, back(d + 1)) + r[1]) + r[2 + j];
                            }
                        }
                    }
                }
                if constexpr (ALIGN) {
                    // the cell's own row, for the NaN class (the beta side's check, here on the alpha side)
                    const float *r = lp + ((int64_t)t * ld + u) * W2;
                    saw_nan |= (r[0] != r[0]) || (u < Un - 1 && r[1] != r[1]);
#pragma unroll
                    for (int j = 0; j < KD; ++j)
                        if (j < D) saw_nan |= r[2 + j] != r[2 + j];
                    int k = kTdtNoPred;
                    v = (t == 0 && u == 0) ? 0.0f : max_cands(c, k);
                    o.dec[base + (int64_t)t * ld + u] = (uint8_t)k;
                } else {
                    v = (t == 0 && u == 0) ? 0.0f : lse_cands(c);
                }
            } else {
                // push-side view: the cell's own weights, beta of the destinations; a blank to t + d == Tn from the
                // last column is terminal (beta 0 after it)
                const float *r = lp + ((int64_t)t * ld + u) * W2;
                const float b = r[0], l = r[1];
                const bool has_label = u < Un - 1;
                saw_nan |= (b != b) || (has_label && l != l);
#pragma unroll
                for (int j = 0; j < KD; ++j) {
                    c[2 * j] = c[2 * j + 1] = -INFINITY;
                    if (j < D) {
                        const int d = a.dur.d[j], tq = t + d;
                        const float ld = r[2 + j];
                        saw_nan |= ld != ld;
                        if (d > 0) {
                            if (tq < Tn) c[2 * j] = (b + ld) + rd(tq, u, fwd(d));
                            else if (tq == Tn && !has_label) c[2 * j] = b + ld;
                        }
                        if (has_label && tq < Tn) c[2 * j + 1] = (l + ld) + rd(tq, u + 1, fwd(d + 1));
                    }
                }
                v = lse_cands(c);
            }
            if (R) ring[slot * U + u] = v;
            out[(int64_t)t * ld + u] = v;
        }
        __syncthreads();
    }
    if (!beta_side && !ALIGN) return;
    bool bad = false;
    for (int u = threadIdx.x; u < Un - 1; u += blockDim.x) {
        const int lab = labels[u];
        bad |= lab < 0 || lab >= a.V;
    }
    bad = __syncthreads_or(bad);
    saw_nan = __syncthreads_or(saw_nan);
    if constexpr (ALIGN && MB) {
        // the terminal step, by the tie rule of max_cands_mb: the standard blank from (Tn - 1, Un - 1), then big blank
        // j from (Tn - d[j], Un - 1) by increasing duration.  Every thread computes it alike, as below.
        float best = -INFINITY;
        int t0 = 0, k0 = kTdtNoPred;
        const int64_t last = (int64_t)(Tn - 1) * ld + Un - 1;
        const float cs = out[last] + lp[last * W2];
        if (cs > best) { best = cs; t0 = Tn - 1; k0 = 0; }
        for (int j = 0; j < D; ++j) {
            const int tp = Tn - a.dur.d[j];
            if (tp >= 0) {
                const int64_t src = (int64_t)tp * ld + Un - 1;
                const float cand = out[src] + lp[src * W2 + 2 + j];
                if (cand > best) { best = cand; t0 = tp; k0 = 2 + j; }
            }
        }
        const int st = bad ? kTdtInvalid : saw_nan ? kTdtNan : lattice_dead(best) ? kTdtDead : kTdtOk;
        if (threadIdx.x == 0) {
            a.status[n] = st;
            a.costs[n] = st == kTdtOk ? best : st == kTdtDead ? -INFINITY : NAN;
        }
        mb_backtrace<KD>(a, o, base, ld, lab_base, COMPACT ? Un - 1 : U - 1, n, Un, t0, k0, st == kTdtOk);
        return;
    } else if constexpr (ALIGN) {
        // the terminal step: the best blank edge of duration d > 0 from (Tn - d, Un - 1), by the tie rule of
        // max_cands (the shorter duration wins).  Every thread computes it alike from alpha in global memory (the
        // sweep ended on a barrier), so the choice needs no broadcast and the ring keeps all of shared memory.
        float best = -INFINITY;
        int t0 = 0;
        for (int j = 0; j < D; ++j) {
            const int d = a.dur.d[j], tp = Tn - d;
            if (d > 0 && tp >= 0) {
                const float *r = lp + ((int64_t)tp * ld + Un - 1) * W2;
                const float cand = (out[(int64_t)tp * ld + Un - 1] + r[0]) + r[2 + j];
                if (cand > best) { best = cand; t0 = tp; }
            }
        }
        const int st = bad ? kTdtInvalid : saw_nan ? kTdtNan : lattice_dead(best) ? kTdtDead : kTdtOk;
        if (threadIdx.x == 0) {
            a.status[n] = st;
            a.costs[n] = st == kTdtOk ? best : st == kTdtDead ? -INFINITY : NAN;
        }
        tdt_backtrace(a, o, base, ld, lab_base, COMPACT ? Un - 1 : U - 1, Tn, Un, t0, st == kTdtOk);
        return;
    }
    if (threadIdx.x == 0) {
        const float lP = out[0];
        const int st = bad ? kTdtInvalid : saw_nan ? kTdtNan : lattice_dead(lP) ? kTdtDead : kTdtOk;
        a.status[n] = st;
        a.ll[n] = lP;
        a.costs[n] = st == kTdtOk ? -lP : st == kTdtDead ? INFINITY : NAN;
    }
}

template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads) k_tdt_recur(TdtRec a) {
    tdt_recur<KD, false>(a, TdtCompact{});
}

// The multi-blank alpha / beta, grid (N, 2): a.D = B, a.dur the big blanks' durations.  One CTA per SM is all the
// bound promises: without it ptxas holds the compact KD = 17 body to 40 registers and spills.
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads, 1) k_mb_recur(TdtRec a) {
    tdt_recur<KD, false, false, true>(a, TdtCompact{});
}
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads, 1) k_mb_recur_compact(TdtRec a, TdtCompact cp) {
    tdt_recur<KD, true, false, true>(a, cp);
}

// The Viterbi alignment, one CTA per lattice (grid (N, 1)): a.costs = the scores; a.beta, a.ll unused
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads) k_tdt_align(TdtRec a, TdtAlignOut o) {
    tdt_recur<KD, false, true>(a, TdtCompact{}, o);
}
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads) k_tdt_align_compact(TdtRec a, TdtCompact cp, TdtAlignOut o) {
    tdt_recur<KD, true, true>(a, cp, o);
}

// The multi-blank Viterbi alignment, grid (N, 1): a.D = B, a.costs = the scores.  The bound of k_mb_recur.
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads, 1) k_mb_align(TdtRec a, MbAlignOut o) {
    tdt_recur<KD, false, true, true>(a, TdtCompact{}, o);
}
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads, 1) k_mb_align_compact(TdtRec a, TdtCompact cp, MbAlignOut o) {
    tdt_recur<KD, true, true, true>(a, cp, o);
}

// a.T, a.U = max_T, max_U
template <int KD>
__global__ void __launch_bounds__(kTdtMaxThreads) k_tdt_recur_compact(TdtRec a, TdtCompact cp) {
    tdt_recur<KD, true>(a, cp);
}

// Edge posteriors per cell: (Pb, Pl, Pd[0..D)), one thread per cell.  0 on padding and on lattices with invalid input
// or no path; NaN on the live cells of a lattice with a NaN (or +inf, or all -inf) live row.  COMPACT: cells = STU, and
// a row that lies in no lattice, or in one that is not ok, is a padding row.  MB: (P_std, Pl, P_big[0..B)), the
// posterior of each of the cell's edges.
template <int KD, bool COMPACT, bool MB = false>
__device__ __forceinline__ void
tdt_post_rows(const float *__restrict__ lp, const float *__restrict__ alpha, const float *__restrict__ beta,
              const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
              const int *__restrict__ yn, int64_t cells, int U, int D, const TdtDurations &dur, FastDiv divU,
              FastDiv divTU, float *__restrict__ pg, const TdtCompact &cp) {
    const int W2 = 2 + D;
    for (int64_t cell = (int64_t)blockIdx.x * kTdtRowThreads + threadIdx.x; cell < cells;
         cell += (int64_t)gridDim.x * kTdtRowThreads) {
        uint32_t n, rem, t, u;
        int Tn, Un, st, rs;                                      // rs: row stride
        bool live;
        float *g = pg + cell * W2;
        if constexpr (COMPACT) {
            const int m = tdt_find(cp.mem_pref, cp.N, cell);
            n = max(m, 0);
            Tn = xn[n]; Un = yn[n] + 1;
            st = m < 0 ? kTdtInvalid : status[n];
            const int64_t local = cell - cp.mem_pref[n];
            live = st != kTdtInvalid && local < (int64_t)Tn * Un;     // an ok lattice: Un >= 1, rows inside STU
            t = live ? (uint32_t)local / (uint32_t)Un : 0;
            u = live ? (uint32_t)local % (uint32_t)Un : 0;
            rs = Un;
        } else {
            divTU.divmod((uint32_t)cell, n, rem);
            divU.divmod(rem, t, u);
            Tn = xn[n]; Un = yn[n] + 1;
            st = status[n];
            live = st != kTdtInvalid && (int)t < Tn && (int)u < Un;   // status Invalid covers bad lengths
            rs = U;
        }
        if (!live || st == kTdtDead || st == kTdtNan) {
            const float z = (live && st == kTdtNan) ? NAN : 0.0f;
            for (int k = 0; k < W2; ++k) g[k] = z;
            continue;
        }
        const float *r = lp + cell * W2;
        const float al = alpha[cell], lP = ll[n], b = r[0], l = r[1];
        const bool has_label = (int)u < Un - 1;
        if constexpr (MB) {
            float ps = 0.0f, pl = 0.0f;
            if ((int)t + 1 < Tn) ps = expf(((al + b) + beta[cell + rs]) - lP);
            else if (!has_label) ps = expf((al + b) - lP);
            if (has_label) pl = expf(((al + l) + beta[cell + 1]) - lP);
            g[0] = ps;
            g[1] = pl;
#pragma unroll
            for (int j = 0; j < KD - 2; ++j) {
                if (j < D) {
                    const int d = dur.d[j], tq = (int)t + d;
                    float pj = 0.0f;
                    if (tq < Tn) pj = expf(((al + r[2 + j]) + beta[cell + (int64_t)d * rs]) - lP);
                    else if (tq == Tn && !has_label) pj = expf((al + r[2 + j]) - lP);
                    g[2 + j] = pj;
                }
            }
            continue;
        }
        float pb = 0.0f, pl = 0.0f;
#pragma unroll
        for (int j = 0; j < KD; ++j) {
            if (j < D) {
                const int d = dur.d[j], tq = (int)t + d;
                const float ld = r[2 + j];
                float gb = 0.0f, gl = 0.0f;
                if (d > 0) {
                    if (tq < Tn) gb = expf((((al + b) + ld) + beta[cell + (int64_t)d * rs]) - lP);
                    else if (tq == Tn && !has_label) gb = expf(((al + b) + ld) - lP);
                }
                if (has_label && tq < Tn) gl = expf((((al + l) + ld) + beta[cell + (int64_t)d * rs + 1]) - lP);
                pb += gb;
                pl += gl;
                g[2 + j] = gb + gl;
            }
        }
        g[0] = pb;
        g[1] = pl;
    }
}

template <int KD>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_post(const float *__restrict__ lp, const float *__restrict__ alpha, const float *__restrict__ beta,
           const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
           const int *__restrict__ yn, int64_t cells, int T, int U, int D, TdtDurations dur, FastDiv divU,
           FastDiv divTU, float *__restrict__ pg) {
    tdt_post_rows<KD, false>(lp, alpha, beta, ll, status, xn, yn, cells, U, D, dur, divU, divTU, pg, TdtCompact{});
}

template <int KD>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_post(const float *__restrict__ lp, const float *__restrict__ alpha, const float *__restrict__ beta,
          const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
          const int *__restrict__ yn, int64_t cells, int T, int U, int D, TdtDurations dur, FastDiv divU,
          FastDiv divTU, float *__restrict__ pg) {
    tdt_post_rows<KD, false, true>(lp, alpha, beta, ll, status, xn, yn, cells, U, D, dur, divU, divTU, pg,
                                   TdtCompact{});
}
template <int KD>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_post_compact(const float *__restrict__ lp, const float *__restrict__ alpha, const float *__restrict__ beta,
                  const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
                  const int *__restrict__ yn, int D, TdtDurations dur, float *__restrict__ pg, TdtCompact cp) {
    tdt_post_rows<KD, true, true>(lp, alpha, beta, ll, status, xn, yn, cp.STU, cp.max_U, D, dur, FastDiv(), FastDiv(),
                                  pg, cp);
}

template <int KD>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_post_compact(const float *__restrict__ lp, const float *__restrict__ alpha, const float *__restrict__ beta,
                   const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
                   const int *__restrict__ yn, int D, TdtDurations dur, float *__restrict__ pg, TdtCompact cp) {
    tdt_post_rows<KD, true>(lp, alpha, beta, ll, status, xn, yn, cp.STU, cp.max_U, D, dur, FastDiv(), FastDiv(), pg,
                            cp);
}

// The row data one gradient element needs.  zero: the row's posteriors are all 0 (padding, no path, or a cell no path
// visits): the row is written as exact zeros and neither the logits nor lse are read.  COMPACT: a row with posteriors
// lies in an ok lattice, found by tdt_find (U, divU and divTU are not used).  MB (LSE = float): occ is the sum of all
// 2 + B posteriors and zero says it is 0 (each is >= 0 or NaN); ld is not used.
struct TdtRow {
    const float *pd;
    float occ, pb, pl, lt, ld, sc;
    int lab;
    bool zero;
};
template <bool COMPACT, bool MB = false, typename LSE = float2>
__device__ __forceinline__ TdtRow tdt_row(int64_t row, const LSE *lse, const float *pg, const int *labels,
                                          const float *grad_out, int U, int W2, const FastDiv &divU,
                                          const FastDiv &divTU, const TdtCompact &cp, const int *yn) {
    TdtRow r;
    r.pd = pg + row * W2;
    r.pb = r.pd[0];
    r.pl = r.pd[1];
    if constexpr (MB) {
        float occ = r.pb + r.pl;
        for (int k = 2; k < W2; ++k) occ += r.pd[k];
        r.occ = occ;
        r.zero = occ == 0.0f;
    } else {
        r.zero = r.pb == 0.0f && r.pl == 0.0f;
        r.occ = r.pb + r.pl;
    }
    r.lt = r.ld = r.sc = 0.0f;
    r.lab = -1;
    if (!r.zero) {
        if constexpr (MB) {
            r.lt = lse[row];
        } else {
            const float2 q = lse[row];
            r.lt = q.x;
            r.ld = q.y;
        }
        if constexpr (COMPACT) {
            const int n = tdt_find(cp.mem_pref, cp.N, row);
            const int Un = yn[n] + 1, u = (int)((uint32_t)(row - cp.mem_pref[n]) % (uint32_t)Un);
            r.lab = (u < Un - 1) ? labels[cp.lab_pref[n] + u] : -1;
            r.sc = grad_out ? grad_out[n] : 1.0f;
        } else {
            uint32_t n, rem, t, u;
            divTU.divmod((uint32_t)row, n, rem);
            divU.divmod(rem, t, u);
            r.lab = ((int)u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : -1;
            r.sc = grad_out ? grad_out[n] : 1.0f;
        }
    }
    return r;
}
__device__ __forceinline__ float tdt_elem(const TdtRow &r, int v, float xv, int V, int blank) {
    if (r.zero) return 0.0f;
    if (v < V) {
        float sel = (v == blank) ? r.pb : 0.0f;
        if (v == r.lab) sel += r.pl;
        return (r.occ * expf(xv - r.lt) - sel) * r.sc;
    }
    return (r.occ * expf(xv - r.ld) - r.pd[2 + (v - V)]) * r.sc;
}
// the multi-blank gradient element of column v < V; big blank j = blank - 1 - v when 0 <= j < B
__device__ __forceinline__ float mb_elem(const TdtRow &r, int v, float xv, int B, int blank) {
    if (r.zero) return 0.0f;
    float sel = (v == blank) ? r.pb : 0.0f;
    const int j = blank - 1 - v;
    if (j >= 0 && j < B) sel += r.pd[2 + j];
    if (v == r.lab) sel += r.pl;
    return (r.occ * expf(xv - r.lt) - sel) * r.sc;
}

// Gradient emit: the flat (rows, W) output in vectors of VEC elements (16 bytes when `out` is 16-byte aligned, else 1),
// which may straddle rows; XVEC: the logits are read with the same vectors (x aligned as out), else element by element.
// Every element is computed the same way whatever VEC, XVEC, the element type and the layout; bf16 is rounded once on
// the store.  COMPACT: the rows are the (STU, W) rows of the compact layout, vectors straddle lattices as they
// straddle rows.  MB: rows of W = V (mb_elem), lse (rows) floats.
template <typename IO, int VEC, bool XVEC, bool COMPACT, bool MB = false, typename LSE = float2>
__device__ __forceinline__ void
tdt_emit_flat(const IO *__restrict__ x, const LSE *__restrict__ lse, const float *__restrict__ pg,
              const int *__restrict__ labels, const float *__restrict__ grad_out, IO *__restrict__ out, int64_t total,
              int V, int D, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows, int stride_v,
              const TdtCompact &cp, const int *__restrict__ yn) {
    const int W = MB ? V : V + D, W2 = 2 + D;
    int64_t f = ((int64_t)blockIdx.x * kTdtRowThreads + threadIdx.x) * VEC;
    if (f >= total) return;
    int64_t row = f / W;
    int v0 = (int)(f - row * W);
    const int64_t stride = stride_rows * W + stride_v;
    auto row_at = [&](int64_t i) {
        return tdt_row<COMPACT, MB>(i, lse, pg, labels, grad_out, U, W2, divU, divTU, cp, yn);
    };
    auto elem = [&](const TdtRow &r, int v, float xv) {
        if constexpr (MB) return mb_elem(r, v, xv, D, blank);
        else return tdt_elem(r, v, xv, V, blank);
    };
    for (; f < total; f += stride, row += stride_rows, v0 += stride_v) {
        if (v0 >= W) { v0 -= W; ++row; }
        float e[VEC];
        TdtRow r = row_at(row);
        if (f + VEC <= total) {
            float xv[VEC];
            const bool whole = v0 + VEC <= W;
            if (XVEC && !(whole && r.zero)) {
                ld_logits<VEC>(x + f, xv);
            } else {
#pragma unroll
                for (int k = 0; k < VEC; ++k) xv[k] = 0.0f;
            }
            int64_t rw = row;
            int v = v0;
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                if (v == W) { v = 0; ++rw; r = row_at(rw); }
                if (!XVEC && !r.zero) xv[k] = io_load(x + f + k);
                e[k] = elem(r, v, xv[k]);
                ++v;
            }
            if constexpr (VEC == 1) st_one(out + f, e[0]);
            else st_vec(out + f, e);
        } else {
            // the last, partial vector of the tensor
            int64_t rw = row;
            int v = v0;
            for (int64_t i = f; i < total; ++i) {
                if (v == W) { v = 0; ++rw; r = row_at(rw); }
                st_one(out + i, elem(r, v, r.zero ? 0.0f : io_load(x + i)));
                ++v;
            }
        }
    }
}

template <typename IO, int VEC, bool XVEC>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_emit(const IO *__restrict__ x, const float2 *__restrict__ lse, const float *__restrict__ pg,
           const int *__restrict__ labels, const float *__restrict__ grad_out, IO *__restrict__ out, int64_t total,
           int V, int D, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows, int stride_v) {
    tdt_emit_flat<IO, VEC, XVEC, false>(x, lse, pg, labels, grad_out, out, total, V, D, blank, U, divU, divTU,
                                        stride_rows, stride_v, TdtCompact{}, nullptr);
}

// total = STU * (V + D)
template <typename IO, int VEC, bool XVEC>
__global__ void __launch_bounds__(kTdtRowThreads)
k_tdt_emit_compact(const IO *__restrict__ x, const float2 *__restrict__ lse, const float *__restrict__ pg,
                   const int *__restrict__ labels, const int *__restrict__ yn, const float *__restrict__ grad_out,
                   IO *__restrict__ out, int64_t total, int V, int D, int blank, int64_t stride_rows, int stride_v,
                   TdtCompact cp) {
    tdt_emit_flat<IO, VEC, XVEC, true>(x, lse, pg, labels, grad_out, out, total, V, D, blank, 0, FastDiv(), FastDiv(),
                                       stride_rows, stride_v, cp, yn);
}

template <typename IO, int VEC, bool XVEC>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_emit(const IO *__restrict__ x, const float *__restrict__ lse, const float *__restrict__ pg,
          const int *__restrict__ labels, const float *__restrict__ grad_out, IO *__restrict__ out, int64_t total,
          int V, int D, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows, int stride_v) {
    tdt_emit_flat<IO, VEC, XVEC, false, true>(x, lse, pg, labels, grad_out, out, total, V, D, blank, U, divU, divTU,
                                              stride_rows, stride_v, TdtCompact{}, nullptr);
}
template <typename IO, int VEC, bool XVEC>
__global__ void __launch_bounds__(kTdtRowThreads)
k_mb_emit_compact(const IO *__restrict__ x, const float *__restrict__ lse, const float *__restrict__ pg,
                  const int *__restrict__ labels, const int *__restrict__ yn, const float *__restrict__ grad_out,
                  IO *__restrict__ out, int64_t total, int V, int D, int blank, int64_t stride_rows, int stride_v,
                  TdtCompact cp) {
    tdt_emit_flat<IO, VEC, XVEC, true, true>(x, lse, pg, labels, grad_out, out, total, V, D, blank, 0, FastDiv(),
                                             FastDiv(), stride_rows, stride_v, cp, yn);
}

// Process-wide, unlike the loss' per-thread record (api.cu): autograd runs the backward on its own device thread, and
// the record must see the emit of the same call.
static std::mutex g_tdt_mu;
static int32_t g_tdt_record[RNNT_TDT_RECORD_LEN];
static int32_t g_tdt_seq;

static int max_optin_smem(int dev) {
    static std::atomic<int> cache[kMaxDevices];
    if (dev < kMaxDevices) { const int c = cache[dev].load(std::memory_order_relaxed); if (c > 0) return c; }
    int b = 48 << 10;
    cudaDeviceGetAttribute(&b, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (dev < kMaxDevices) cache[dev].store(b, std::memory_order_relaxed);
    return b;
}

void tdt_launch_record(int32_t *out) {
    std::lock_guard<std::mutex> lock(g_tdt_mu);
    memcpy(out, g_tdt_record, sizeof(g_tdt_record));
}

TdtPlan tdt_plan(int U, const TdtDurations &dur, const void *x, int elem_bytes, int V, bool multiblank) {
    TdtPlan p;
    const int W = multiblank ? V : V + dur.D;
    const int eoff = (int)((reinterpret_cast<uintptr_t>(x) / (uintptr_t)elem_bytes) & 3u);   // element alignment
    p.norm_group = (W % 4 == 0 && eoff == 0) ? 4 : (W % 2 == 0 && (eoff & 1) == 0) ? 2 : 1;
    p.norm_lanes = W <= 64 ? 8 : 32;
    // TDT: D candidate pairs; multi-blank: 2 + B candidates
    p.kd = (multiblank ? 2 + dur.D : dur.D) <= 5 ? 5 : kTdtMaxD;
    p.warps = min((U + 31) / 32, kTdtMaxThreads / 32);
    p.passes = (U + p.warps * 32 - 1) / (p.warps * 32);
    p.ring = dur.dmax + (multiblank ? 1 : 2);
    const int64_t smem = (int64_t)p.ring * U * (int64_t)sizeof(float);
    if (smem > max_optin_smem(current_device())) p.ring = 0;
    p.smem = p.ring ? (int)smem : 0;
    return p;
}

// the compact layout of a forward (c.mem_pref set)
static TdtCompact tdt_compact(const TdtFwd &c) { return {c.mem_pref, c.lab_pref, c.STU, c.N, c.T, c.U}; }

template <bool MB, typename IN>
static cudaError_t tdt_norm_as(cudaStream_t s, const TdtPlan &p, const IN *x, const TdtFwd &c, int64_t cells) {
    // the dense cell -> (n, t, u) divisions (the compact kernels find lattices through mem_pref instead)
    const FastDiv divU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)c.U);
    const FastDiv divTU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)(c.T * c.U));
    const int64_t per_block = kTdtRowThreads / p.norm_lanes;
    const unsigned grid = (unsigned)min((cells + per_block - 1) / per_block, (int64_t)sm_count(current_device()) * 16);
    // compact: CTA rows per lattice as logits.cu's compact normaliser sizes them
    const dim3 cgrid(compact_gx(cells, c.N, per_block * kCompactIters), c.N);
#define RNNT_TDT_NORM(SUB, G)                                                                                         \
    if constexpr (MB) {                                                                                               \
        if (c.mem_pref)                                                                                               \
            k_mb_norm_compact<IN, SUB, G><<<cgrid, kTdtRowThreads, 0, s>>>(x, c.labels, c.xn, c.yn, c.V, c.dur.D,     \
                                                                           c.blank, c.sigma, c.lse_mb, c.lp,          \
                                                                           tdt_compact(c));                           \
        else                                                                                                          \
            k_mb_norm<IN, SUB, G><<<grid, kTdtRowThreads, 0, s>>>(x, c.labels, c.xn, c.yn, cells, c.T, c.U, c.V,      \
                                                                  c.dur.D, c.blank, c.sigma, divU, divTU, c.lse_mb,   \
                                                                  c.lp);                                              \
    } else                                                                                                            \
    (c.mem_pref                                                                                                       \
         ? k_tdt_norm_compact<IN, SUB, G><<<cgrid, kTdtRowThreads, 0, s>>>(x, c.labels, c.xn, c.yn, c.V, c.dur.D,     \
                                                                           c.blank, c.sigma, c.lse, c.lp,             \
                                                                           tdt_compact(c))                            \
         : k_tdt_norm<IN, SUB, G><<<grid, kTdtRowThreads, 0, s>>>(x, c.labels, c.xn, c.yn, cells, c.T, c.U, c.V,      \
                                                                  c.dur.D, c.blank, c.sigma, divU, divTU, c.lse, c.lp))
    if (p.norm_lanes == 8) {
        if (p.norm_group == 4) { RNNT_TDT_NORM(8, 4); } else if (p.norm_group == 2) { RNNT_TDT_NORM(8, 2); } else { RNNT_TDT_NORM(8, 1); }
    } else {
        if (p.norm_group == 4) { RNNT_TDT_NORM(32, 4); } else if (p.norm_group == 2) { RNNT_TDT_NORM(32, 2); } else { RNNT_TDT_NORM(32, 1); }
    }
#undef RNNT_TDT_NORM
    count_launch();
    return cudaGetLastError();
}

template <int KD, bool MB>
static cudaError_t tdt_recur_post(cudaStream_t s, const TdtPlan &p, const TdtFwd &c, int64_t cells) {
    static std::atomic<bool> smem_set[kMaxDevices], smem_set_compact[kMaxDevices];
    const auto recur = MB ? k_mb_recur<KD> : k_tdt_recur<KD>;
    const auto recur_compact = MB ? k_mb_recur_compact<KD> : k_tdt_recur_compact<KD>;
    if (p.smem > (48 << 10)) {
        const cudaError_t e = c.mem_pref ? ensure_dyn_smem(recur_compact, smem_set_compact,
                                                           max_optin_smem(current_device()))
                                         : ensure_dyn_smem(recur, smem_set, max_optin_smem(current_device()));
        if (e != cudaSuccess) return e;
    }
    TdtRec r = {c.lp, c.labels, c.xn, c.yn, c.alpha, c.beta, c.ll, c.costs, c.status, c.T, c.U, c.V, c.dur.D, p.ring,
                c.dur};
    if (c.mem_pref) recur_compact<<<dim3(c.N, 2), p.warps * 32, p.smem, s>>>(r, tdt_compact(c));
    else recur<<<dim3(c.N, 2), p.warps * 32, p.smem, s>>>(r);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || !c.pg || cells == 0) return e;
    // the dense cell -> (n, t, u) divisions (the compact kernels find lattices through mem_pref instead)
    const FastDiv divU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)c.U);
    const FastDiv divTU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)(c.T * c.U));
    const unsigned grid = (unsigned)min((cells + kTdtRowThreads - 1) / kTdtRowThreads,
                                        (int64_t)sm_count(current_device()) * 16);
    const auto post = MB ? k_mb_post<KD> : k_tdt_post<KD>;
    const auto post_compact = MB ? k_mb_post_compact<KD> : k_tdt_post_compact<KD>;
    if (c.mem_pref)
        post_compact<<<grid, kTdtRowThreads, 0, s>>>(c.lp, c.alpha, c.beta, c.ll, c.status, c.xn, c.yn, c.dur.D, c.dur,
                                                     c.pg, tdt_compact(c));
    else
        post<<<grid, kTdtRowThreads, 0, s>>>(c.lp, c.alpha, c.beta, c.ll, c.status, c.xn, c.yn, cells, c.T, c.U,
                                             c.dur.D, c.dur, divU, divTU, c.pg);
    count_launch();
    return cudaGetLastError();
}

// The plan of a forward or alignment call, recorded for rnnt_b200_debug_last_tdt_launch (the emit fields 0)
static TdtPlan tdt_plan_recorded(const TdtFwd &c) {
    const TdtPlan p = tdt_plan(c.U, c.dur, c.x, c.io_bf16 ? 2 : 4, c.V, c.multiblank);
    std::lock_guard<std::mutex> lock(g_tdt_mu);
    int32_t *rec = g_tdt_record;
    memset(rec, 0, sizeof(g_tdt_record));
    rec[RNNT_TDT_REC_SEQ] = ++g_tdt_seq;
    rec[RNNT_TDT_REC_CLUSTER] = 0;
    rec[RNNT_TDT_REC_WARPS] = p.warps;
    rec[RNNT_TDT_REC_RING] = p.ring;
    rec[RNNT_TDT_REC_PASSES] = p.passes;
    rec[RNNT_TDT_REC_KD] = p.kd;
    rec[RNNT_TDT_REC_NORM_GROUP] = p.norm_group;
    rec[RNNT_TDT_REC_NORM_LANES] = p.norm_lanes;
    rec[RNNT_TDT_REC_SMEM] = p.smem;
    return p;
}

cudaError_t launch_tdt_forward(cudaStream_t s, const TdtFwd &c) {
    const int64_t cells = c.mem_pref ? c.STU : (int64_t)c.N * c.T * c.U;
    const TdtPlan p = tdt_plan_recorded(c);
    if (cells == 0 && !c.mem_pref) return cudaSuccess;   // compact: with no rows the recurrence still gives the costs
    if (c.multiblank) {
        const cudaError_t e = c.io_bf16 ? tdt_norm_as<true>(s, p, static_cast<const __nv_bfloat16 *>(c.x), c, cells)
                                        : tdt_norm_as<true>(s, p, static_cast<const float *>(c.x), c, cells);
        if (e != cudaSuccess) return e;
        return p.kd == 5 ? tdt_recur_post<5, true>(s, p, c, cells) : tdt_recur_post<kTdtMaxD, true>(s, p, c, cells);
    }
    cudaError_t e = c.io_bf16 ? tdt_norm_as<false>(s, p, static_cast<const __nv_bfloat16 *>(c.x), c, cells)
                              : tdt_norm_as<false>(s, p, static_cast<const float *>(c.x), c, cells);
    if (e != cudaSuccess) return e;
    return p.kd == 5 ? tdt_recur_post<5, false>(s, p, c, cells) : tdt_recur_post<kTdtMaxD, false>(s, p, c, cells);
}

template <int KD>
static cudaError_t tdt_align_as(cudaStream_t s, const TdtPlan &p, const TdtFwd &c, const TdtAlignOut &o) {
    static std::atomic<bool> smem_set[kMaxDevices], smem_set_compact[kMaxDevices];
    if (p.smem > (48 << 10)) {
        const cudaError_t e = c.mem_pref ? ensure_dyn_smem(k_tdt_align_compact<KD>, smem_set_compact,
                                                           max_optin_smem(current_device()))
                                         : ensure_dyn_smem(k_tdt_align<KD>, smem_set, max_optin_smem(current_device()));
        if (e != cudaSuccess) return e;
    }
    const TdtRec r = {c.lp, c.labels, c.xn, c.yn, c.alpha, nullptr, nullptr, c.costs, c.status, c.T, c.U, c.V,
                      c.dur.D, p.ring, c.dur};
    if (c.mem_pref) k_tdt_align_compact<KD><<<dim3(c.N, 1), p.warps * 32, p.smem, s>>>(r, tdt_compact(c), o);
    else k_tdt_align<KD><<<dim3(c.N, 1), p.warps * 32, p.smem, s>>>(r, o);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_tdt_align(cudaStream_t s, const TdtFwd &c, uint8_t *dec, int *frames, int *fdur) {
    const int64_t cells = c.mem_pref ? c.STU : (int64_t)c.N * c.T * c.U;
    const TdtPlan p = tdt_plan_recorded(c);
    cudaError_t e = c.io_bf16 ? tdt_norm_as<false>(s, p, static_cast<const __nv_bfloat16 *>(c.x), c, cells)
                              : tdt_norm_as<false>(s, p, static_cast<const float *>(c.x), c, cells);
    if (e != cudaSuccess) return e;
    const TdtAlignOut o = {dec, frames, fdur};
    return p.kd == 5 ? tdt_align_as<5>(s, p, c, o) : tdt_align_as<kTdtMaxD>(s, p, c, o);
}

template <int KD>
static cudaError_t mb_align_as(cudaStream_t s, const TdtPlan &p, const TdtFwd &c, const MbAlignOut &o) {
    static std::atomic<bool> smem_set[kMaxDevices], smem_set_compact[kMaxDevices];
    if (p.smem > (48 << 10)) {
        const cudaError_t e = c.mem_pref ? ensure_dyn_smem(k_mb_align_compact<KD>, smem_set_compact,
                                                           max_optin_smem(current_device()))
                                         : ensure_dyn_smem(k_mb_align<KD>, smem_set, max_optin_smem(current_device()));
        if (e != cudaSuccess) return e;
    }
    const TdtRec r = {c.lp, c.labels, c.xn, c.yn, c.alpha, nullptr, nullptr, c.costs, c.status, c.T, c.U, c.V,
                      c.dur.D, p.ring, c.dur};
    if (c.mem_pref) k_mb_align_compact<KD><<<dim3(c.N, 1), p.warps * 32, p.smem, s>>>(r, tdt_compact(c), o);
    else k_mb_align<KD><<<dim3(c.N, 1), p.warps * 32, p.smem, s>>>(r, o);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_mb_align(cudaStream_t s, const TdtFwd &c, uint8_t *dec, int *frames, int *counts) {
    const int64_t cells = c.mem_pref ? c.STU : (int64_t)c.N * c.T * c.U;
    const TdtPlan p = tdt_plan_recorded(c);
    cudaError_t e = c.io_bf16 ? tdt_norm_as<true>(s, p, static_cast<const __nv_bfloat16 *>(c.x), c, cells)
                              : tdt_norm_as<true>(s, p, static_cast<const float *>(c.x), c, cells);
    if (e != cudaSuccess) return e;
    const MbAlignOut o = {dec, frames, counts};
    return p.kd == 5 ? mb_align_as<5>(s, p, c, o) : mb_align_as<kTdtMaxD>(s, p, c, o);
}

template <bool MB, typename IO>
static cudaError_t tdt_emit_as(cudaStream_t s, const TdtBwd &c, const IO *x, IO *out) {
    const int W = MB ? c.V : c.V + c.D;
    const int64_t total = (c.mem_pref ? c.STU : (int64_t)c.N * c.T * c.U) * W;
    constexpr int kVec = 16 / (int)sizeof(IO);
    const bool ovec = (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
    const bool xvec = ovec && (reinterpret_cast<uintptr_t>(x) & 15u) == 0;
    const int vec = ovec ? kVec : 1;
    {
        std::lock_guard<std::mutex> lock(g_tdt_mu);
        g_tdt_record[RNNT_TDT_REC_EMIT_VEC] = vec;
        g_tdt_record[RNNT_TDT_REC_EMIT_XVEC] = xvec;
    }
    if (total == 0) return cudaSuccess;
    // the dense cell -> (n, t, u) divisions (the compact kernels find lattices through mem_pref instead)
    const FastDiv divU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)c.U);
    const FastDiv divTU = c.mem_pref ? FastDiv() : FastDiv((uint32_t)(c.T * c.U));
    const int64_t vecs = (total + vec - 1) / vec;
    const unsigned grid = (unsigned)min((vecs + kTdtRowThreads - 1) / kTdtRowThreads,
                                        (int64_t)sm_count(current_device()) * 32);
    const int64_t stride = (int64_t)grid * kTdtRowThreads * vec;
    const int64_t srows = stride / W;
    const int sv = (int)(stride - srows * W);
    const TdtCompact cp = {c.mem_pref, c.lab_pref, c.STU, c.N, 0, 0};
#define RNNT_TDT_EMIT(VEC, XV)                                                                                        \
    if constexpr (MB) {                                                                                               \
        if (c.mem_pref)                                                                                               \
            k_mb_emit_compact<IO, VEC, XV><<<grid, kTdtRowThreads, 0, s>>>(x, c.lse_mb, c.pg, c.labels, c.yn,         \
                                                                           c.grad_out, out, total, c.V, c.D, c.blank, \
                                                                           srows, sv, cp);                            \
        else                                                                                                          \
            k_mb_emit<IO, VEC, XV><<<grid, kTdtRowThreads, 0, s>>>(x, c.lse_mb, c.pg, c.labels, c.grad_out, out,      \
                                                                   total, c.V, c.D, c.blank, c.U, divU, divTU, srows, \
                                                                   sv);                                               \
    } else                                                                                                            \
    (c.mem_pref                                                                                                       \
         ? k_tdt_emit_compact<IO, VEC, XV><<<grid, kTdtRowThreads, 0, s>>>(x, c.lse, c.pg, c.labels, c.yn, c.grad_out, \
                                                                           out, total, c.V, c.D, c.blank, srows, sv,  \
                                                                           cp)                                        \
         : k_tdt_emit<IO, VEC, XV><<<grid, kTdtRowThreads, 0, s>>>(x, c.lse, c.pg, c.labels, c.grad_out, out, total,  \
                                                                   c.V, c.D, c.blank, c.U, divU, divTU, srows, sv))
    if (!ovec) { RNNT_TDT_EMIT(1, false); }
    else if (xvec) { RNNT_TDT_EMIT(kVec, true); }
    else { RNNT_TDT_EMIT(kVec, false); }
#undef RNNT_TDT_EMIT
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_tdt_backward(cudaStream_t s, const TdtBwd &c) {
    if (c.multiblank) {
        if (c.io_bf16)
            return tdt_emit_as<true>(s, c, static_cast<const __nv_bfloat16 *>(c.x), static_cast<__nv_bfloat16 *>(c.out));
        return tdt_emit_as<true>(s, c, static_cast<const float *>(c.x), static_cast<float *>(c.out));
    }
    if (c.io_bf16)
        return tdt_emit_as<false>(s, c, static_cast<const __nv_bfloat16 *>(c.x), static_cast<__nv_bfloat16 *>(c.out));
    return tdt_emit_as<false>(s, c, static_cast<const float *>(c.x), static_cast<float *>(c.out));
}

}  // namespace rnnt
