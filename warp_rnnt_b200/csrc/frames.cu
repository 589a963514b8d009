// frames.cu -- the one-symbol-per-frame lattices of k2 (rnnt_type "modified" and "constrained") and the delay penalty,
// both on the f32 (N,T,U,2) (blank, label) pairs that every k2-family forward produces (include/rnnt_b200.h gives the
// semantics and the classes of degenerate input).
//
//   k_delay_pairs  one elementwise pass: l += ((Tn-1)/2 - t) * lambda at every live label slot (k2's delay_penalty)
//   k_frames       alpha (blockIdx.y = 0) and beta (1) of lattice blockIdx.x.  Under the modified lattice both edges
//                  leave the frame, so row t+1 depends on row t only: the sweep runs by frame (Tn steps, each reading
//                  one contiguous pair row) with the lattice's columns spread over the CTA's threads; the previous
//                  row sits in shared memory (two row buffers).  The beta CTA classifies the lattice and writes its cost.
//   k_frames_grads one thread per cell: d cost / d (blank, label) in the (N,T,U,2) pair_grads convention of the regular
//                  path, so that every backward kernel consumes them unchanged.  Constrained: the label weight is
//                  l(t,u) + b(t,u+1), so the label edge's occupation is also added to the blank slot of (t,u+1); the
//                  blank slot before that fold can be written on its own for the prune ranges.
//   k_frames_align k_frames' alpha side in max-plus form, with one decision word per warp and frame, then the
//                  backtrace in the same CTA: the Viterbi alignment on these lattices (rnnt_b200_align_logits_dense).
//
// Every operand is clamped below at kBig (a -inf log-prob becomes the finite sentinel) and every LSE is the exact
// max + log1pf(expf(-|d|)) of two finite values or NaN, so -inf - -inf is never formed; a lattice with no finite path
// ends with beta[0,0] at about kBig.  No atomics: every value has one writer and a fixed operation order.
#include <cstring>

#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kFramesMaxThreads = 512;   // k_frames: threads over the columns, a thread takes every blockDim-th column
constexpr int kFramesGradThreads = 256;
constexpr int kDelayThreads = 256;

// lattice classes, written by the beta CTA into the workspace's status (N)
enum { kFramesOk = 0, kFramesInvalid = 1, kFramesNan = 2, kFramesDead = 3 };

__device__ __forceinline__ float fr_clamp(float v) { return v < kBig ? kBig : v; }   // NaN stays NaN
__device__ __forceinline__ float fr_lse(float a, float b) {
    return fmaxf(a, b) + log1pf(expf(-fabsf(a - b)));                               // NaN in, NaN out
}

__device__ __forceinline__ bool fr_lengths(const int *xn, const int *yn, int n, int T, int U, int &Tn, int &Un) {
    Tn = xn[n];
    Un = yn[n] + 1;
    return Tn >= 1 && Tn <= T && Un >= 1 && Un <= U;
}

// pairs_out[cell] = pairs_in[cell], with the penalty added to the label of every live label slot (t < Tn, u < Un-1
// of a lattice with valid lengths), in f32 in the stated order; in place when the two are the same.
__global__ void __launch_bounds__(kDelayThreads)
k_delay_pairs(const float2 *pairs_in, float2 *pairs_out, const int *__restrict__ xn, const int *__restrict__ yn,
              uint32_t cells, int T, int U, FastDiv divU, FastDiv divTU, float lam) {
    for (uint32_t cell = blockIdx.x * kDelayThreads + threadIdx.x; cell < cells; cell += gridDim.x * kDelayThreads) {
        uint32_t n, rem, t, u;
        divTU.divmod(cell, n, rem);
        divU.divmod(rem, t, u);
        int Tn, Un;
        float2 w = pairs_in[cell];
        if (fr_lengths(xn, yn, (int)n, T, U, Tn, Un) && (int)t < Tn && (int)u < Un - 1) {
            const float pen = __fmul_rn(__fsub_rn(__fmul_rn((float)(Tn - 1), 0.5f), (float)t), lam);
            w.y = __fadd_rn(w.y, pen);
        }
        pairs_out[cell] = w;
    }
}

struct FramesArgs {
    const float2 *pairs;
    const int *xn, *yn;
    float *alphas, *betas, *ll, *costs;
    int *status;
    int T, U;
};

// alpha(0,0) = 0, alpha(0,u>0) = kBig; alpha(t+1,u) = LSE(alpha(t,u) + b(t,u), alpha(t,u-1) + l'(t,u-1)), where
// l'(t,u) = l(t,u) (+ b(t,u+1) constrained).  beta(Tn,u) = 0 at u = Un-1, kBig elsewhere;
// beta(t,u) = LSE(b(t,u) + beta(t+1,u), l'(t,u) + beta(t+1,u+1)), the label term absent on the last column.
// A step's pair operands do not depend on the recurrence: those of the thread's first kFramesPrefetch columns are
// loaded one frame ahead into registers, so that their latency overlaps the step before; further columns (U > 1024)
// are loaded in their step.
constexpr int kFramesPrefetch = 2;

// the raw pair operands of column u in a step: alpha side (b(t,u), l(t,u-1)), beta side (b(t,u), l(t,u), b(t,u+1))
struct FrOps { float b, l, b1; };
template <bool BETA, bool CONSTRAINED>
__device__ __forceinline__ FrOps fr_ops(const float2 *row, int u, int Un) {
    FrOps o;
    o.b = __ldg(&row[u].x);
    o.l = o.b1 = 0.0f;
    if (!BETA && u > 0) o.l = __ldg(&row[u - 1].y);
    if (BETA && u < Un - 1) {
        o.l = __ldg(&row[u].y);
        if (CONSTRAINED) o.b1 = __ldg(&row[u + 1].x);
    }
    return o;
}

template <bool CONSTRAINED>
__global__ void __launch_bounds__(kFramesMaxThreads) k_frames(FramesArgs a) {
    extern __shared__ float rows[];                 // two row buffers of a.U floats
    const int n = blockIdx.x;
    const bool beta_side = blockIdx.y == 1;
    int Tn, Un;
    if (!fr_lengths(a.xn, a.yn, n, a.T, a.U, Tn, Un)) {
        if (beta_side && threadIdx.x == 0) {
            a.status[n] = kFramesInvalid;
            a.ll[n] = NAN;
            a.costs[n] = NAN;
        }
        return;
    }
    const int U = a.U, bd = blockDim.x;
    const int64_t base = (int64_t)n * a.T * U;
    const float2 *pr = a.pairs + base;
    auto buf = [&](int t) { return rows + (t & 1) * U; };   // the row buffer of frame t
    FrOps pf[kFramesPrefetch];
    bool saw_nan = false;
    if (!beta_side) {
        float *out = a.alphas + base;
        for (int u = threadIdx.x; u < Un; u += bd) {
            const float v = u == 0 ? 0.0f : kBig;
            buf(0)[u] = v;
            out[u] = v;
        }
#pragma unroll
        for (int k = 0; k < kFramesPrefetch; ++k)
            if (threadIdx.x + k * bd < Un && Tn > 1)
                pf[k] = fr_ops<false, CONSTRAINED>(pr, threadIdx.x + k * bd, Un);
        __syncthreads();
        for (int t = 1; t < Tn; ++t) {
            const float *prev = buf(t - 1);
            float *cur = buf(t);
            const float2 *row = pr + (int64_t)(t - 1) * U;
            auto step = [&](int u, const FrOps &o) {
                const float b = fr_clamp(o.b);
                const float vb = prev[u] + b;
                float v = vb;
                if (u > 0) {
                    float l = fr_clamp(o.l);
                    if (CONSTRAINED) l = l + b;
                    v = fr_lse(vb, prev[u - 1] + l);
                }
                cur[u] = v;
                out[(int64_t)t * U + u] = v;
            };
#pragma unroll
            for (int k = 0; k < kFramesPrefetch; ++k) {
                const int u = threadIdx.x + k * bd;
                if (u < Un) {
                    const FrOps o = pf[k];
                    if (t + 1 < Tn) pf[k] = fr_ops<false, CONSTRAINED>(row + U, u, Un);
                    step(u, o);
                }
            }
            for (int u = threadIdx.x + kFramesPrefetch * bd; u < Un; u += bd)
                step(u, fr_ops<false, CONSTRAINED>(row, u, Un));
            __syncthreads();
        }
        return;
    }
    float *out = a.betas + base;
    for (int u = threadIdx.x; u < Un; u += bd) buf(Tn)[u] = (u == Un - 1) ? 0.0f : kBig;
#pragma unroll
    for (int k = 0; k < kFramesPrefetch; ++k)
        if (threadIdx.x + k * bd < Un)
            pf[k] = fr_ops<true, CONSTRAINED>(pr + (int64_t)(Tn - 1) * U, threadIdx.x + k * bd, Un);
    __syncthreads();
    for (int t = Tn - 1; t >= 0; --t) {
        const float *nxt = buf(t + 1);
        float *cur = buf(t);
        const float2 *row = pr + (int64_t)t * U;
        auto step = [&](int u, const FrOps &o) {
            saw_nan |= (o.b != o.b) || (o.l != o.l);
            const float b = fr_clamp(o.b);
            float v = b + nxt[u];
            if (u < Un - 1) {
                float l = fr_clamp(o.l);
                if (CONSTRAINED) l = l + fr_clamp(o.b1);
                v = fr_lse(v, l + nxt[u + 1]);
            }
            cur[u] = v;
            out[(int64_t)t * U + u] = v;
        };
#pragma unroll
        for (int k = 0; k < kFramesPrefetch; ++k) {
            const int u = threadIdx.x + k * bd;
            if (u < Un) {
                const FrOps o = pf[k];
                if (t > 0) pf[k] = fr_ops<true, CONSTRAINED>(row - U, u, Un);
                step(u, o);
            }
        }
        for (int u = threadIdx.x + kFramesPrefetch * bd; u < Un; u += bd)
            step(u, fr_ops<true, CONSTRAINED>(row, u, Un));
        __syncthreads();
    }
    saw_nan = __syncthreads_or(saw_nan);
    if (threadIdx.x == 0) {
        const float lP = buf(0)[0];
        const int st = saw_nan ? kFramesNan : lattice_dead(lP) ? kFramesDead : kFramesOk;
        a.status[n] = st;
        a.ll[n] = lP;
        a.costs[n] = st == kFramesOk ? -lP : st == kFramesDead ? INFINITY : NAN;
    }
}

// Viterbi alignment on the modified / constrained lattice (rnnt_b200_align_logits_dense, rnnt_type 1 or 2): alpha in
// max-plus form, alpha(0,0) = 0, alpha(0,u>0) = -inf, alpha(t+1,u) = skip = alpha(t,u) + b(t,u), or emit =
// alpha(t,u-1) + l'(t,u-1) iff emit > skip or skip is NaN (column 0: skip).  The weights are not clamped: max-plus
// never subtracts, so -inf stays -inf.  The sweep and its operand prefetch are k_frames' alpha side, one frame per
// step; each warp also stores the __ballot_sync of its 32 columns' choices as one word of dec (N, ceil(U/32), T), so
// that one coalesced load serves 32 frames of a column block.  Then warp 0 walks the path back from (Tn, Un-1): the
// walk leaves one frame per step and at most one column, so 32 steps need the words of the current column block and
// of the one to its left; those of the next 32 frames are loaded while the walk runs on shuffled copies.
struct FramesAlignArgs {
    const float2 *pairs;
    const int *xn, *yn;
    uint32_t *dec;
    float *scores;
    int *frames;                    // (N, U-1)
    int T, U;
};

template <bool CONSTRAINED>
__global__ void __launch_bounds__(kFramesMaxThreads) k_frames_align(FramesAlignArgs a) {
    extern __shared__ float rows[];                 // two row buffers of a.U floats
    const int n = blockIdx.x;
    const int U = a.U, bd = blockDim.x, lane = threadIdx.x & 31;
    int *fr = a.frames + (int64_t)n * (U - 1);
    int Tn, Un;
    const bool ok = fr_lengths(a.xn, a.yn, n, a.T, U, Tn, Un);
    if (!ok || Un - 1 > Tn) {                       // invalid lengths: NaN; more labels than frames: no path, -inf
        for (int u = threadIdx.x; u < U - 1; u += bd) fr[u] = -1;
        if (threadIdx.x == 0) a.scores[n] = ok ? -INFINITY : NAN;
        return;
    }
    const float2 *pr = a.pairs + (int64_t)n * a.T * U;
    uint32_t *dec = a.dec + (int64_t)n * ((U + 31) >> 5) * a.T;
    auto buf = [&](int t) { return rows + (t & 1) * U; };   // the row buffer of frame t
    for (int u = threadIdx.x; u < Un; u += bd) buf(0)[u] = u == 0 ? 0.0f : -INFINITY;
    FrOps pf[kFramesPrefetch];
#pragma unroll
    for (int k = 0; k < kFramesPrefetch; ++k)
        if (threadIdx.x + k * bd < Un) pf[k] = fr_ops<false, CONSTRAINED>(pr, threadIdx.x + k * bd, Un);
    __syncthreads();
    for (int t = 0; t < Tn; ++t) {
        const float *prev = buf(t);
        float *cur = buf(t + 1);
        const float2 *row = pr + (int64_t)t * U;
        auto step = [&](int u, const FrOps &o) {
            const float skip = prev[u] + o.b;
            bool e = false;
            float v = skip;
            if (u > 0) {
                const float emit = prev[u - 1] + (CONSTRAINED ? o.l + o.b : o.l);
                e = emit > skip || isnan(skip);
                if (e) v = emit;
            }
            cur[u] = v;
            return e;
        };
        // u0: the warp's first column (warp-uniform), below Un
        auto store = [&](int u0, bool e) {
            const unsigned word = __ballot_sync(0xffffffffu, e);
            if (lane == 0) dec[(int64_t)(u0 >> 5) * a.T + t] = word;
        };
#pragma unroll
        for (int k = 0; k < kFramesPrefetch; ++k) {
            const int u = threadIdx.x + k * bd;
            if (u - lane < Un) {
                bool e = false;
                if (u < Un) {
                    const FrOps o = pf[k];
                    if (t + 1 < Tn) pf[k] = fr_ops<false, CONSTRAINED>(row + U, u, Un);
                    e = step(u, o);
                }
                store(u - lane, e);
            }
        }
        for (int u0 = threadIdx.x - lane + kFramesPrefetch * bd; u0 < Un; u0 += bd) {
            const int u = u0 + lane;
            store(u0, u < Un && step(u, fr_ops<false, CONSTRAINED>(row, u, Un)));
        }
        __syncthreads();
    }
    if (threadIdx.x >= 32) return;
    const float score = buf(Tn)[Un - 1];
    const bool live = score > -INFINITY;            // -inf: no path above -inf; NaN: every path NaN
    for (int u = (live ? Un - 1 : 0) + lane; u < U - 1; u += 32) fr[u] = -1;
    if (lane == 0) a.scores[n] = score;
    if (!live) return;
    // Backtrace over chunks of 32 frames: lane k holds the words of frame s_hi - k of column blocks w (cur) and w - 1
    // (left); ul is the column inside block w, negative once the walk has entered block w - 1.  Lane k keeps its
    // step's column and bit and writes that label's frame after the chunk.  Frames below 0 read as zero words.
    auto ld = [&](int blk, int s) -> uint32_t {
        return (blk >= 0 && s - lane >= 0) ? dec[(int64_t)blk * a.T + s - lane] : 0u;
    };
    int u = Un - 1, s_hi = Tn - 1, w = u >> 5;
    uint32_t cur = ld(w, s_hi), left = ld(w - 1, s_hi);
    while (true) {
        const int s_next = s_hi - 32;
        const uint32_t ncur = ld(w, s_next), nleft = ld(w - 1, s_next);
        int ul = u - 32 * w, my_u = 0, my_b = 0;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const uint32_t wc = __shfl_sync(0xffffffffu, cur, k), wl = __shfl_sync(0xffffffffu, left, k);
            const int b = (int)(((ul >= 0 ? wc : wl) >> (ul & 31)) & 1u);
            if (lane == k) { my_u = 32 * w + ul; my_b = b; }
            ul -= b;
        }
        if (my_b) fr[my_u - 1] = s_hi - lane;       // label edge (t, my_u - 1) -> (t + 1, my_u)
        u = 32 * w + ul;
        if (s_next < 0) break;
        s_hi = s_next;
        if (ul < 0) {                               // entered block w - 1: its words are the prefetched left ones
            --w;
            cur = nleft;
            left = ld(w - 1, s_hi);
        } else {
            cur = ncur;
            left = nleft;
        }
    }
}

// occupation of the label edge out of (t,u), u < Un-1: exp(alpha + l' + beta(t+1,u+1) - ll), with beta(Tn,Un-1) = 0
// and no edge into (Tn, u+1 < Un-1)
template <bool CONSTRAINED>
__device__ __forceinline__ float fr_label_occ(const float2 *pairs, const float *alphas, const float *betas, int64_t cell,
                                              int t, int u, int Tn, int Un, int U, float lP) {
    float l = fr_clamp(pairs[cell].y);
    if (CONSTRAINED) l = l + fr_clamp(pairs[cell + 1].x);
    float nb;
    if (t + 1 < Tn) nb = betas[cell + U + 1];
    else if (u + 1 == Un - 1) nb = 0.0f;
    else return 0.0f;
    return expf(((alphas[cell] + l) + nb) - lP);
}

// pair_grads (N,T,U,2): every cell written.  raw: (N,T,U) blank slots before the constrained fold, or null.
template <bool CONSTRAINED>
__global__ void __launch_bounds__(kFramesGradThreads)
k_frames_grads(const float2 *__restrict__ pairs, const float *__restrict__ alphas, const float *__restrict__ betas,
               const float *__restrict__ ll, const int *__restrict__ status, const int *__restrict__ xn,
               const int *__restrict__ yn, uint32_t cells, int U, FastDiv divU, FastDiv divTU,
               float2 *__restrict__ pg, float *__restrict__ raw) {
    for (uint32_t cell = blockIdx.x * kFramesGradThreads + threadIdx.x; cell < cells;
         cell += gridDim.x * kFramesGradThreads) {
        uint32_t n, rem, t, u;
        divTU.divmod(cell, n, rem);
        divU.divmod(rem, t, u);
        const int st = status[n];
        const int Tn = xn[n], Un = yn[n] + 1;
        const bool live = st != kFramesInvalid && (int)t < Tn && (int)u < Un;
        float gb = 0.0f, gl = 0.0f, rb = 0.0f;
        if (live && st == kFramesNan) {
            gb = rb = NAN;
            gl = (int)u < Un - 1 ? NAN : 0.0f;
        } else if (live && st == kFramesOk) {
            const float lP = ll[n];
            float nb = 0.0f;
            bool edge = true;
            if ((int)t + 1 < Tn) nb = betas[cell + U];
            else edge = (int)u == Un - 1;
            const float ob = edge ? expf(((alphas[cell] + fr_clamp(pairs[cell].x)) + nb) - lP) : 0.0f;
            rb = -ob;
            gb = rb;
            if ((int)u < Un - 1)
                gl = -fr_label_occ<CONSTRAINED>(pairs, alphas, betas, cell, t, u, Tn, Un, U, lP);
            if (CONSTRAINED && u > 0)
                gb = gb - fr_label_occ<CONSTRAINED>(pairs, alphas, betas, cell - 1, t, u - 1, Tn, Un, U, lP);
        }
        pg[cell] = make_float2(gb, gl);
        if (raw) raw[cell] = rb;
    }
}

static thread_local int32_t t_frames_record[RNNT_FRAMES_RECORD_LEN];
static thread_local int32_t t_frames_seq;
void frames_launch_record(int32_t *out) { memcpy(out, t_frames_record, sizeof(t_frames_record)); }

static int grid_for(uint32_t cells, int threads) {
    const int64_t want = ((int64_t)cells + threads - 1) / threads;
    return (int)max((int64_t)1, min(want, (int64_t)sm_count(current_device()) * 16));
}

cudaError_t launch_delay_pairs(cudaStream_t s, const float2 *pairs_in, float2 *pairs_out, const int *xn, const int *yn,
                               int N, int T, int U, float lam) {
    const uint32_t cells = (uint32_t)((int64_t)N * T * U);
    k_delay_pairs<<<grid_for(cells, kDelayThreads), kDelayThreads, 0, s>>>(
        pairs_in, pairs_out, xn, yn, cells, T, U, FastDiv((uint32_t)U), FastDiv((uint32_t)T * (uint32_t)U), lam);
    count_launch();
    return cudaGetLastError();
}

size_t frames_smem_bytes(int U) { return 2 * (size_t)U * sizeof(float); }

template <bool C>
static cudaError_t launch_frames_c(cudaStream_t s, const FramesCall &c) {
    static std::atomic<bool> attr_done[kMaxDevices];
    const cudaError_t e = ensure_dyn_smem(k_frames<C>, attr_done, (int)frames_smem_bytes(kFramesMaxU));
    if (e != cudaSuccess) return e;
    const int threads = min(kFramesMaxThreads, max(32, (c.U + 31) / 32 * 32));
    const size_t smem = frames_smem_bytes(c.U);
    FramesArgs a = {c.pairs, c.xn, c.yn, c.alphas, c.betas, c.ll, c.costs, c.status, c.T, c.U};
    k_frames<C><<<dim3(c.N, 2), threads, smem, s>>>(a);
    count_launch();
    const uint32_t cells = (uint32_t)((int64_t)c.N * c.T * c.U);
    const int gx = grid_for(cells, kFramesGradThreads);
    if (c.pair_grads) {
        k_frames_grads<C><<<gx, kFramesGradThreads, 0, s>>>(c.pairs, c.alphas, c.betas, c.ll, c.status, c.xn, c.yn,
                                                             cells, c.U, FastDiv((uint32_t)c.U),
                                                             FastDiv((uint32_t)c.T * (uint32_t)c.U), c.pair_grads,
                                                             c.raw_blank);
        count_launch();
    }
    int32_t *rec = t_frames_record;
    rec[RNNT_FRAMES_REC_SEQ] = ++t_frames_seq;
    rec[RNNT_FRAMES_REC_CONSTRAINED] = C;
    rec[RNNT_FRAMES_REC_THREADS] = threads;
    rec[RNNT_FRAMES_REC_PASSES] = (c.U + threads - 1) / threads;
    rec[RNNT_FRAMES_REC_SMEM] = (int32_t)smem;
    rec[RNNT_FRAMES_REC_GRAD_BLOCKS] = c.pair_grads ? gx : 0;
    return cudaGetLastError();
}

cudaError_t launch_frames(cudaStream_t s, const FramesCall &c, bool delayed) {
    memset(t_frames_record, 0, sizeof(t_frames_record));
    t_frames_record[RNNT_FRAMES_REC_DELAY] = delayed;
    return c.constrained ? launch_frames_c<true>(s, c) : launch_frames_c<false>(s, c);
}

static thread_local int32_t t_frames_align_record[RNNT_FRAMES_ALIGN_RECORD_LEN];
static thread_local int32_t t_frames_align_seq;
void frames_align_launch_record(int32_t *out) {
    memcpy(out, t_frames_align_record, sizeof(t_frames_align_record));
}

template <bool C>
static cudaError_t launch_frames_align_c(cudaStream_t s, const FramesAlignCall &c) {
    static std::atomic<bool> attr_done[kMaxDevices];
    const cudaError_t e = ensure_dyn_smem(k_frames_align<C>, attr_done, (int)frames_smem_bytes(kFramesMaxU));
    if (e != cudaSuccess) return e;
    const int threads = min(kFramesMaxThreads, max(32, (c.U + 31) / 32 * 32));
    const size_t smem = frames_smem_bytes(c.U);
    FramesAlignArgs a = {c.pairs, c.xn, c.yn, c.dec, c.scores, c.frames, c.T, c.U};
    k_frames_align<C><<<c.N, threads, smem, s>>>(a);
    count_launch();
    int32_t *rec = t_frames_align_record;
    memset(rec, 0, sizeof(t_frames_align_record));
    rec[RNNT_FRAMES_ALIGN_REC_SEQ] = ++t_frames_align_seq;
    rec[RNNT_FRAMES_ALIGN_REC_CONSTRAINED] = C;
    rec[RNNT_FRAMES_ALIGN_REC_THREADS] = threads;
    rec[RNNT_FRAMES_ALIGN_REC_PASSES] = (c.U + threads - 1) / threads;
    rec[RNNT_FRAMES_ALIGN_REC_SMEM] = (int32_t)smem;
    rec[RNNT_FRAMES_ALIGN_REC_BLOCKS] = (c.U + 31) / 32;
    rec[RNNT_FRAMES_ALIGN_REC_DELAY] = c.delayed;
    return cudaGetLastError();
}

cudaError_t launch_frames_align(cudaStream_t s, const FramesAlignCall &c) {
    return c.constrained ? launch_frames_align_c<true>(s, c) : launch_frames_align_c<false>(s, c);
}

}  // namespace rnnt
