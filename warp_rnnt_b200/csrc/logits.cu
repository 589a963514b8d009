// logits.cu -- the step BEFORE the reference's path, fused in: the loss straight from un-normalised joint-network
// logits (SURVEY.md 8(f)1).
//
// The reference requires log-softmaxed input (the reference's README.md:59) and its benchmark times F.log_softmax with
// the loss (pytorch_binding/benchmark.py:65): log_softmax forward (read + write of (N,T,U,V)), the loss (read + dense
// gradient write, + mul_) and log_softmax backward (two reads + one write) -- seven dense passes.  Here:
//
//   k_lse_pairs      one read of the logits: per cell the normaliser lse = max + log(sum exp(x - max)) and the two
//                    normalised log-probs the recurrence needs, pairs[cell] = (x[blank] - lse, x[label] - lse)
//   (wavefront)      the existing kernels on the (cells,2) layout -> (cells,2) gradients w.r.t. the log-probs
//   k_expand_logits  one read of the logits + one write: the gradient w.r.t. the LOGITS,
//                        g[v] = [v == blank] gb + [v == label] gl - exp(x[v] - lse) (gb + gl),
//                    i.e. log_softmax's backward applied to the loss' (blank, label) gradient on the fly, times grad_out[n]
//
// three dense passes in total.  A label equal to blank: the two gradients add (what autograd through torch.gather /
// log_softmax does).  Padded cells carry zero pair gradients and get exact zeros (NaN where the row's normaliser is
// NaN, as log_softmax's backward gives).
//
// Both dense kernels take float or bf16 logits (SURVEY.md 8(f)2); the bf16 gradient is bf16 too.  Everything between
// the load and the store is fp32 and the same for both types: k_lse_pairs sums a bf16 row in the order it sums the
// float row of the same V (same SUB, same lanes, same groups of 4 -- a bf16 group is one 8-byte load where a float
// group is a float4), so lse and pairs are bit for bit those of the float path on the widened logits; k_expand_logits
// computes every element as the float kernel does and rounds it to bf16 once, on the store.
//
// HAT (the Hybrid Autoregressive Transducer's normalisation, k2's get_hat_logprobs): the same passes with a second
// normalisation, a template flag on the row bodies, instantiated as kernels of their own (k_*_hat) so the softmax
// kernels stay exactly as they are.  The blank is a sigmoid and the labels a softmax over the non-blank columns:
//   lse   = lse_nb, the normaliser of the row with column B excluded by index (summed as a row whose x[B] is -inf)
//   pairs = (logsigmoid(x[B]), x[y] - lse_nb + logsigmoid(-x[B])), logsigmoid(z) = min(z, 0) - log1p(exp(-|z|))
//   grad  = gl ([v == y] - exp(x[v] - lse_nb)) at v != B, gb sigmoid(-x[B]) - gl sigmoid(x[B]) (+ gl if y == B) at B
// and a row with pair gradients (0, 0) gets zeros, NaN at v != B when lse_nb is NaN and at B when x[B] is NaN.
#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kLogitThreads = 256;

// group q of 4 consecutive logits of a row whose groups are aligned (4 * sizeof(IN) bytes)
__device__ __forceinline__ float4 ld_group4(const float *row, int q) { return __ldg(reinterpret_cast<const float4 *>(row) + q); }
__device__ __forceinline__ float4 ld_group4(const __nv_bfloat16 *row, int q) {
    const uint2 r = __ldg(reinterpret_cast<const uint2 *>(row) + q);
    return make_float4(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u), __uint_as_float(r.y << 16),
                       __uint_as_float(r.y & 0xffff0000u));
}

// SUB lanes cooperate on one cell (SUB in {1, 8, 32}); online max / sum so the row is read once.  VEC4: rows are whole
// groups of 4 at group-aligned addresses -> the SUB lanes stride over groups (float V = 28: 7 of 8 lanes load one float4
// each, a warp reads 4 consecutive rows = 448 contiguous bytes).  The choice of SUB and VEC4 depends on V and the
// alignment only, never on IN: a bf16 row is summed exactly like the float row of the same values.
//
// COMPACT: the rows are joint_pack's ragged (STU, V) order and the grid is (gx, N): CTA row blockIdx.y streams over the
// Tn*Un rows of lattice n (Problem `lay`, compact prefix sums), the pointers rebased to its first row.  Only the
// (lattice, u, label) of a row differs from the dense kernel; a row is summed exactly as the dense row of its values.
//
// PRUNED (ROWS == kRowsPruned): the rows are rnnt_loss_pruned's (N,T,S,V) windows; row (n,t,s) is cell (t, u) of the
// full (N,T,U) lattice with u = ranges[n,t] + s (divU divides by S, divTU by T).  lse is written for every row, the
// pair only for 0 <= u < U, at that cell of the full (N,T,U,2) pairs; k_fill_pairs gave every other cell
// (kBig, kBig) before.  Again only the mapping differs: a row is summed exactly as the dense row of its values.
enum { kRowsDense = 0, kRowsCompact = 1, kRowsPruned = 2 };

// HAT: group q of a row with its element at column `blank` (if any) set to -inf, as the sums read it
__device__ __forceinline__ float4 hat_group4(float4 a, int q, int blank) {
    const int k = blank - 4 * q;
    a.x = k == 0 ? -INFINITY : a.x;
    a.y = k == 1 ? -INFINITY : a.y;
    a.z = k == 2 ? -INFINITY : a.z;
    a.w = k == 3 ? -INFINITY : a.w;
    return a;
}

// HAT: the (blank, label) log-probs of a row from its non-blank normaliser l, in the order include/rnnt_b200.h states
template <typename IN>
__device__ __forceinline__ float2 hat_pair(const IN *row, int blank, int lab, float l) {
    const float xb = io_load(row + blank), sp = log1pf(expf(-fabsf(xb)));
    return make_float2(fminf(xb, 0.0f) - sp, (io_load(row + lab) - l) + (fminf(-xb, 0.0f) - sp));
}

template <typename IN, int SUB, bool VEC4, int ROWS, bool HAT = false>
__device__ __forceinline__ void
lse_pairs_rows(const IN *__restrict__ x, const int *__restrict__ labels, int64_t cells, int V, int blank, int U,
               FastDiv divU, FastDiv divTU, float2 *__restrict__ pairs, float *__restrict__ lse_out, Problem lay,
               const int *__restrict__ ranges) {
    constexpr bool COMPACT = ROWS == kRowsCompact;
    Lattice L;
    if constexpr (COMPACT) {
        // `cells` = STU on entry: a lattice never reaches past the rows of the tensor (lengths the hints vouched for)
        L = get_lattice(lay, blockIdx.y);
        cells = L.ok ? max(min((int64_t)L.Tn * L.Un, cells - L.base), (int64_t)0) : 0;
        x += L.base * V; pairs += L.base; lse_out += L.base;
    }
    const int sub = threadIdx.x % SUB;
    const int64_t per_block = kLogitThreads / SUB;
    for (int64_t base = (int64_t)blockIdx.x * per_block; base < cells; base += (int64_t)gridDim.x * per_block) {   // block-uniform trip count
        const int64_t cell = min(base + threadIdx.x / SUB, cells - 1);          // surplus groups redo the last cell (shuffles need every lane)
        const IN *row = x + cell * V;
        float m = -INFINITY, s = 0.0f;
        // The online sums below subtract the running max m, which stays -inf while every logit seen so far is -inf
        // (a masked vocabulary entry): exp(-inf - (-inf)) would be NaN.  Until a finite logit arrives they subtract 0
        // instead -- exp(-inf) = 0, and a NaN logit still makes the sum NaN; with a finite m nothing changes.
        auto off = [&]() { return m == -INFINITY ? 0.0f : m; };
        auto add = [&](float a) {
            if (a > m) { s = s * expf(m - a); m = a; }        // (m == -inf: s is 0 or NaN, exp(-inf) = 0)
            s += expf(a - off());
        };
        if (VEC4 && (V >> 2) <= SUB) {
            // the whole row is one group per lane: max first (shuffles only), then ONE exp per element -- the online
            // merge below would spend two more exp per lane and shuffle round
            const bool has = sub < (V >> 2);
            if constexpr (HAT) {
                // (the softmax branch below with the blank masked; kept apart so that branch compiles as it did)
                const float4 a = hat_group4(
                    has ? ld_group4(row, sub) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), sub, blank);
                m = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
#pragma unroll
                for (int o = SUB / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                s = has ? (expf(a.x - m) + expf(a.y - m)) + (expf(a.z - m) + expf(a.w - m)) : 0.0f;
            } else {
                const float4 a = has ? ld_group4(row, sub) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
                m = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
#pragma unroll
                for (int o = SUB / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                s = has ? (expf(a.x - m) + expf(a.y - m)) + (expf(a.z - m) + expf(a.w - m)) : 0.0f;
            }
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        } else if (VEC4 && HAT) {
            // only the group that holds the blank is masked: one lane, one iteration, the selects loop-invariant
            const int qb = blank >> 2;
            for (int q = sub; q < (V >> 2); q += SUB) {
                float4 a = ld_group4(row, q);
                if (q == qb) a = hat_group4(a, qb, blank);
                const float mx = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
                if (mx > m) { s = s * expf(m - mx); m = mx; }
                const float mo = off();
                s += (expf(a.x - mo) + expf(a.y - mo)) + (expf(a.z - mo) + expf(a.w - mo));
            }
        } else if (VEC4) {
            for (int q = sub; q < (V >> 2); q += SUB) {
                const float4 a = ld_group4(row, q);
                const float mx = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
                if (mx > m) { s = s * expf(m - mx); m = mx; }
                const float mo = off();
                s += (expf(a.x - mo) + expf(a.y - mo)) + (expf(a.z - mo) + expf(a.w - mo));
            }
        } else if (SUB == 1) {
            // short unaligned rows: one thread per cell; neighbouring threads' rows share cache lines, so the pass over
            // v is served from L1 after the first touch
            if constexpr (HAT) {
                for (int v = 0; v < V; ++v) m = fmaxf(m, v == blank ? -INFINITY : io_load(row + v));
                for (int v = 0; v < V; ++v) s += expf((v == blank ? -INFINITY : io_load(row + v)) - m);
            } else {
                for (int v = 0; v < V; ++v) m = fmaxf(m, io_load(row + v));
                for (int v = 0; v < V; ++v) s += expf(io_load(row + v) - m);
            }
        } else {
            for (int v = sub; v < V; v += SUB) add(HAT && v == blank ? -INFINITY : io_load(row + v));
        }
        if (SUB > 1 && !(VEC4 && (V >> 2) <= SUB)) {
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
                const float mm = fmaxf(m, m2);
                s = (m == mm ? s : s * expf(m - mm)) + (m2 == mm ? s2 : s2 * expf(m2 - mm));
                m = mm;
            }
        }
        if (sub == 0) {
            // every logit -inf: NaN, as torch.log_softmax gives (and as the max-first paths above compute it)
            const float l = (m == -INFINITY) ? NAN : m + logf(s);
            int lab;
            if constexpr (ROWS == kRowsPruned) {
                uint32_t nt, srow;                               // row = nt * S + srow, nt = n * T + t
                divU.divmod((uint32_t)cell, nt, srow);
                const uint32_t n = divTU.div(nt);
                const int64_t u = (int64_t)ranges[nt] + srow;
                lse_out[cell] = l;
                if (u >= 0 && u < U) {
                    lab = (u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : blank;
                    if constexpr (HAT) pairs[(int64_t)nt * U + u] = hat_pair(row, blank, lab, l);
                    else pairs[(int64_t)nt * U + u] = make_float2(io_load(row + blank) - l, io_load(row + lab) - l);
                }
                continue;
            } else if constexpr (COMPACT) {
                const int u = (int)cell % L.Un;
                lab = (u < L.Un - 1) ? labels[L.lab_base + u] : blank;
            } else {
                uint32_t n, rem, t, u;
                divTU.divmod((uint32_t)cell, n, rem);
                divU.divmod(rem, t, u);
                lab = ((int)u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : blank;
            }
            if constexpr (HAT) pairs[cell] = hat_pair(row, blank, lab, l);
            else pairs[cell] = make_float2(io_load(row + blank) - l, io_load(row + lab) - l);
            lse_out[cell] = l;
        }
    }
}

template <typename IN, int SUB, bool VEC4, bool COMPACT = false>
__global__ void __launch_bounds__(kLogitThreads)
k_lse_pairs(const IN *__restrict__ x, const int *__restrict__ labels, int64_t cells, int V, int blank, int U,
            FastDiv divU, FastDiv divTU, float2 *__restrict__ pairs, float *__restrict__ lse_out, Problem lay) {
    lse_pairs_rows<IN, SUB, VEC4, COMPACT ? kRowsCompact : kRowsDense>(x, labels, cells, V, blank, U, divU, divTU,
                                                                       pairs, lse_out, lay, nullptr);
}

// rows = N*T*S pruned rows; divS, divT: FastDiv(S), FastDiv(T)
template <typename IN, int SUB, bool VEC4>
__global__ void __launch_bounds__(kLogitThreads)
k_lse_pairs_pruned(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ ranges,
                   int64_t rows, int V, int blank, int U, FastDiv divS, FastDiv divT, float2 *__restrict__ pairs,
                   float *__restrict__ lse_out) {
    lse_pairs_rows<IN, SUB, VEC4, kRowsPruned>(x, labels, rows, V, blank, U, divS, divT, pairs, lse_out, Problem{},
                                               ranges);
}

// the HAT twins of k_lse_pairs and k_lse_pairs_pruned (ROWS: kRowsDense, kRowsCompact or kRowsPruned)
template <typename IN, int SUB, bool VEC4, int ROWS>
__global__ void __launch_bounds__(kLogitThreads)
k_lse_pairs_hat(const IN *__restrict__ x, const int *__restrict__ labels, const int *__restrict__ ranges, int64_t cells,
                int V, int blank, int U, FastDiv divU, FastDiv divTU, float2 *__restrict__ pairs,
                float *__restrict__ lse_out, Problem lay) {
    lse_pairs_rows<IN, SUB, VEC4, ROWS, true>(x, labels, cells, V, blank, U, divU, divTU, pairs, lse_out, lay, ranges);
}

// every cell of the full (cells,2) pairs (kBig, kBig): an edge out of a cell that no window row covers is removed
__global__ void __launch_bounds__(kLogitThreads) k_fill_pairs(float4 *__restrict__ pairs2, int64_t cells) {
    const float4 big = make_float4(kBig, kBig, kBig, kBig);
    const int64_t quads = cells >> 1;
    for (int64_t i = (int64_t)blockIdx.x * kLogitThreads + threadIdx.x; i < quads; i += (int64_t)gridDim.x * kLogitThreads)
        pairs2[i] = big;
    if ((cells & 1) && blockIdx.x == 0 && threadIdx.x == 0)
        reinterpret_cast<float2 *>(pairs2)[cells - 1] = make_float2(kBig, kBig);
}

template <int VEC>
__device__ __forceinline__ void st_logit_grads(float *p, const float (&e)[VEC]) {
    if constexpr (VEC == 4) st_cs_v4(p, make_float4(e[0], e[1], e[2], e[3]));
    else if constexpr (VEC == 2) st_cs_v2(p, make_float2(e[0], e[1]));
    else st_cs(p, e[0]);
}
// bf16: every element rounded once (round to nearest even), streaming stores of the vector's width
template <int VEC>
__device__ __forceinline__ void st_logit_grads(__nv_bfloat16 *p, const float (&e)[VEC]) {
    if constexpr (VEC == 8) {
        st_vec(p, e);
    } else if constexpr (VEC == 1) {
        const unsigned short h = __bfloat16_as_ushort(__float2bfloat16_rn(e[0]));
        asm volatile("st.global.cs.b16 [%0], %1;" ::"l"(p), "h"(h) : "memory");
    } else {
        uint32_t w[VEC / 2];
#pragma unroll
        for (int k = 0; k < VEC / 2; ++k) {
            const __nv_bfloat162 h = __floats2bfloat162_rn(e[2 * k], e[2 * k + 1]);
            w[k] = *reinterpret_cast<const uint32_t *>(&h);
        }
        if constexpr (VEC == 4)
            asm volatile("st.global.cs.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(w[0]), "r"(w[1]) : "memory");
        else
            asm volatile("st.global.cs.b32 [%0], %1;" ::"l"(p), "r"(w[0]) : "memory");
    }
}

// flat stream of the (cells, V) output in vectors of VEC elements (float: 4 when V % 4 == 0, 2 when V % 2 == 0, else
// 1; bf16 also 8): a vector never straddles a row, so one (gb, gl, lse, label) fetch serves it.  IO is the element
// type of the logits and of the gradient.  COMPACT: as in k_lse_pairs, CTA row blockIdx.y streams over the Tn*Un*V
// elements of lattice n.
// PRUNED: the rows are the (N,T,S,V) windows, divU divides by S and divTU by T as in k_lse_pairs; row (n,t,s) takes
// (gb, gl) from the full (N,T,U,2) pair gradients at cell (t, u = ranges[n,t] + s), and a row with u outside [0, U) is
// a padding row (pair gradients (0, 0)).
template <typename IO, int VEC, int ROWS, bool HAT = false>
__device__ __forceinline__ void
expand_logits_rows(const IO *__restrict__ x, const float *__restrict__ lse, const float2 *__restrict__ pg,
                   const int *__restrict__ labels, const float *__restrict__ grad_out, IO *__restrict__ out,
                   int64_t cells, int V, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows,
                   int stride_v, const Problem &lay, const int *__restrict__ ranges) {
    constexpr bool COMPACT = ROWS == kRowsCompact;
    Lattice L;
    if constexpr (COMPACT) {
        L = get_lattice(lay, blockIdx.y);
        cells = L.ok ? max(min((int64_t)L.Tn * L.Un, cells - L.base), (int64_t)0) : 0;
        x += L.base * V; out += L.base * V; lse += L.base; pg += L.base;
    }
    const int64_t total = cells * (int64_t)V;
    int64_t f = ((int64_t)blockIdx.x * kLogitThreads + threadIdx.x) * VEC;
    if (f >= total) return;
    // (row, v0) of the thread's vector: one 64-bit division here, then a running cursor (the grid stride is
    // stride_rows whole rows + stride_v elements)
    int64_t row = f / V;
    int v0 = (int)(f - row * V);
    const int64_t stride = stride_rows * V + stride_v;
    for (; f < total; f += stride, row += stride_rows, v0 += stride_v) {
        if (v0 >= V) { v0 -= V; ++row; }
        float2 q;
        int64_t u;                                           // PRUNED: the row's lattice column
        uint32_t nt;                                         // PRUNED: n*T + t
        if constexpr (ROWS == kRowsPruned) {
            uint32_t s;
            divU.divmod((uint32_t)row, nt, s);
            u = (int64_t)ranges[nt] + s;
            q = (u >= 0 && u < U) ? pg[(int64_t)nt * U + u] : make_float2(0.0f, 0.0f);
        } else {
            q = pg[row];
        }
        float e[VEC];
        if (q.x == 0.0f && q.y == 0.0f) {
            // padding (or a cell without gradient): exact zeros -- (0 - softmax * 0), as log_softmax's backward gives,
            // which is NaN when the row's normaliser is NaN (a NaN or +inf logit, or every logit -inf)
            const float z = (lse[row] == lse[row]) ? 0.0f : NAN;
#pragma unroll
            for (int k = 0; k < VEC; ++k) e[k] = z;
            if constexpr (HAT) {
                // HAT: the blank column's normaliser is its own logit (0 * sigmoid(x[B]))
                if ((unsigned)(blank - v0) < (unsigned)VEC) {
                    const float xb = io_load(x + f + (blank - v0));
#pragma unroll
                    for (int k = 0; k < VEC; ++k)
                        if (v0 + k == blank) e[k] = (xb == xb) ? 0.0f : NAN;
                }
            }
        } else {
            int lab;
            float sc;
            if constexpr (ROWS == kRowsPruned) {
                const uint32_t n = divTU.div(nt);
                lab = (u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : -1;
                sc = grad_out ? grad_out[n] : 1.0f;
            } else if constexpr (COMPACT) {
                const int u = (int)row % L.Un;
                lab = (u < L.Un - 1) ? labels[L.lab_base + u] : -1;
                sc = grad_out ? grad_out[blockIdx.y] : 1.0f;
            } else {
                uint32_t n, rem, t, u;
                divTU.divmod((uint32_t)row, n, rem);
                divU.divmod(rem, t, u);
                lab = ((int)u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : -1;
                sc = grad_out ? grad_out[n] : 1.0f;
            }
            const float l = lse[row], tot = q.x + q.y;
            float xv[VEC];
            ld_logits<VEC>(x + f, xv);
            if constexpr (HAT) {
                // the others: log_softmax's backward over v != B for gl; the blank (at most one per vector, computed
                // once outside the unrolled loop): gb sigmoid(-x[B]) - gl sigmoid(x[B])
                float eb = 0.0f;
                if ((unsigned)(blank - v0) < (unsigned)VEC) {
                    const float xb = io_load(x + f + (blank - v0));
                    const float r = expf(-fabsf(xb)), big = 1.0f / (1.0f + r), small = r * big;
                    const bool pos = xb >= 0.0f;
                    eb = ((blank == lab ? q.y : 0.0f) + (q.x * (pos ? small : big) - q.y * (pos ? big : small))) * sc;
                }
#pragma unroll
                for (int k = 0; k < VEC; ++k) {
                    const float gsel = (v0 + k == lab) ? q.y : 0.0f;
                    e[k] = (v0 + k == blank) ? eb : (gsel - expf(xv[k] - l) * q.y) * sc;
                }
            } else {
#pragma unroll
                for (int k = 0; k < VEC; ++k) {
                    float gsel = (v0 + k == blank) ? q.x : 0.0f;
                    if (v0 + k == lab) gsel += q.y;
                    e[k] = (gsel - expf(xv[k] - l) * tot) * sc;
                }
            }
        }
        st_logit_grads<VEC>(out + f, e);
    }
}

template <typename IO, int VEC, bool COMPACT = false>
__global__ void __launch_bounds__(kLogitThreads)
k_expand_logits(const IO *__restrict__ x, const float *__restrict__ lse, const float2 *__restrict__ pg,
                const int *__restrict__ labels, const float *__restrict__ grad_out, IO *__restrict__ out,
                int64_t cells, int V, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows,
                int stride_v, Problem lay) {
    expand_logits_rows<IO, VEC, COMPACT ? kRowsCompact : kRowsDense>(x, lse, pg, labels, grad_out, out, cells, V, blank,
                                                                     U, divU, divTU, stride_rows, stride_v, lay,
                                                                     nullptr);
}

// rows = N*T*S pruned rows, written (N,T,S,V); pg: the full (N,T,U,2) pair gradients; divS, divT: FastDiv(S), FastDiv(T)
template <typename IO, int VEC>
__global__ void __launch_bounds__(kLogitThreads)
k_expand_logits_pruned(const IO *__restrict__ x, const float *__restrict__ lse, const float2 *__restrict__ pg,
                       const int *__restrict__ labels, const int *__restrict__ ranges, const float *__restrict__ grad_out,
                       IO *__restrict__ out, int64_t rows, int V, int blank, int U, FastDiv divS, FastDiv divT,
                       int64_t stride_rows, int stride_v) {
    expand_logits_rows<IO, VEC, kRowsPruned>(x, lse, pg, labels, grad_out, out, rows, V, blank, U, divS, divT,
                                             stride_rows, stride_v, Problem{}, ranges);
}

// the HAT twin of k_expand_logits and k_expand_logits_pruned (ROWS: kRowsDense, kRowsCompact or kRowsPruned)
template <typename IO, int VEC, int ROWS>
__global__ void __launch_bounds__(kLogitThreads)
k_expand_logits_hat(const IO *__restrict__ x, const float *__restrict__ lse, const float2 *__restrict__ pg,
                    const int *__restrict__ labels, const int *__restrict__ ranges, const float *__restrict__ grad_out,
                    IO *__restrict__ out, int64_t cells, int V, int blank, int U, FastDiv divU, FastDiv divTU,
                    int64_t stride_rows, int stride_v, Problem lay) {
    expand_logits_rows<IO, VEC, ROWS, true>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU,
                                            stride_rows, stride_v, lay, ranges);
}

// compact grids: compact_gx (kernels.cuh)
// lay == nullptr: dense (N,T,U,V) logits; else the compact (STU,V) rows of lattices lay->N, lay->T = lay->U = 0.
// ranges != nullptr: the pruned (N,T,S,V) rows of windows ranges (N,T) on the full (N,T,U) lattice.
template <typename IN>
static cudaError_t lse_pairs_as(cudaStream_t s, const IN *x, const int *labels, int N, int T, int U, int V, int blank,
                                float2 *pairs, float *lse, const Problem *lay, int64_t STU, const int *ranges,
                                int S, bool hat) {
    const int64_t cells = lay ? STU : (int64_t)N * T * (ranges ? S : U);
    if (cells <= 0 || N <= 0) return cudaSuccess;
    // pruned: the row -> (n*T + t, s) -> (n, t) divisions
    const FastDiv divU((uint32_t)max(ranges ? S : U, 1)), divTU((uint32_t)max(ranges ? T : T * U, 1));
    const int sms = sm_count(current_device());
    if (ranges) {
        const int64_t quads = (int64_t)N * T * U / 2 + 1;
        k_fill_pairs<<<(unsigned)min((quads + kLogitThreads - 1) / kLogitThreads, (int64_t)sms * 16), kLogitThreads, 0,
                       s>>>(reinterpret_cast<float4 *>(pairs), (int64_t)N * T * U);
        count_launch();
    }
    // groups of 4 elements: float4 (16 bytes) or 4 bf16 (8 bytes) per load
    const bool vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & (4 * sizeof(IN) - 1)) == 0);
    const int sub = vec4 ? (V <= 32 ? 8 : 32) : (V <= 12 ? 1 : (V <= 512 ? 8 : 32));
    const int64_t per_block = kLogitThreads / sub;
    const Problem p = lay ? *lay : Problem{};
    const dim3 grid = lay ? dim3(compact_gx(STU, N, per_block * kCompactIters), N)
                          : dim3((unsigned)min((cells + per_block - 1) / per_block, (int64_t)sms * 16));
#define RNNT_LSE_LAUNCH(SUB, VEC)                                                                                          \
    (hat ? (lay ? k_lse_pairs_hat<IN, SUB, VEC, kRowsCompact><<<grid, kLogitThreads, 0, s>>>(x, labels, ranges, cells, V, blank, U, divU, divTU, pairs, lse, p) \
            : ranges ? k_lse_pairs_hat<IN, SUB, VEC, kRowsPruned><<<grid, kLogitThreads, 0, s>>>(x, labels, ranges, cells, V, blank, U, divU, divTU, pairs, lse, p) \
                : k_lse_pairs_hat<IN, SUB, VEC, kRowsDense><<<grid, kLogitThreads, 0, s>>>(x, labels, ranges, cells, V, blank, U, divU, divTU, pairs, lse, p)) \
     : lay ? k_lse_pairs<IN, SUB, VEC, true><<<grid, kLogitThreads, 0, s>>>(x, labels, cells, V, blank, U, divU, divTU, pairs, lse, p) \
     : ranges ? k_lse_pairs_pruned<IN, SUB, VEC><<<grid, kLogitThreads, 0, s>>>(x, labels, ranges, cells, V, blank, U, divU, divTU, pairs, lse) \
         : k_lse_pairs<IN, SUB, VEC><<<grid, kLogitThreads, 0, s>>>(x, labels, cells, V, blank, U, divU, divTU, pairs, lse, p))
    if (vec4) { if (sub == 8) RNNT_LSE_LAUNCH(8, true); else RNNT_LSE_LAUNCH(32, true); }
    else if (sub == 1) RNNT_LSE_LAUNCH(1, false);
    else if (sub == 8) RNNT_LSE_LAUNCH(8, false);
    else RNNT_LSE_LAUNCH(32, false);
#undef RNNT_LSE_LAUNCH
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_lse_pairs(cudaStream_t s, const void *x, const int *labels, int N, int T, int U, int V, int blank,
                             float2 *pairs, float *lse, int io_bf16, int hat) {
    if (io_bf16)
        return lse_pairs_as(s, static_cast<const __nv_bfloat16 *>(x), labels, N, T, U, V, blank, pairs, lse, nullptr, 0,
                            nullptr, 0, hat);
    return lse_pairs_as(s, static_cast<const float *>(x), labels, N, T, U, V, blank, pairs, lse, nullptr, 0, nullptr, 0,
                        hat);
}

cudaError_t launch_lse_pairs_compact(cudaStream_t s, const void *x, const Problem &p, const int *labels, int64_t STU,
                                     int V, int blank, float2 *pairs, float *lse, int io_bf16, int hat) {
    if (io_bf16)
        return lse_pairs_as(s, static_cast<const __nv_bfloat16 *>(x), labels, p.N, 0, 0, V, blank, pairs, lse, &p, STU,
                            nullptr, 0, hat);
    return lse_pairs_as(s, static_cast<const float *>(x), labels, p.N, 0, 0, V, blank, pairs, lse, &p, STU, nullptr, 0,
                        hat);
}

// lay, ranges: as for lse_pairs_as
template <typename IO>
static cudaError_t expand_logits_as(cudaStream_t s, const IO *x, const float *lse, const float2 *pg, const int *labels,
                                    const float *grad_out, IO *out, int N, int T, int U, int V, int blank,
                                    const Problem *lay, int64_t STU, const int *ranges, int S, bool hat) {
    const int64_t cells = lay ? STU : (int64_t)N * T * (ranges ? S : U);
    if (cells <= 0 || N <= 0) return cudaSuccess;
    const FastDiv divU((uint32_t)max(ranges ? S : U, 1)), divTU((uint32_t)max(ranges ? T : T * U, 1));
    const int sms = sm_count(current_device());
    // the widest vector (at most 16 bytes) that V and the alignment of both tensors allow
    const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out);
    const int vmax = 16 / (int)sizeof(IO);
    int vec = 1;
    for (int c = vmax; c > 1; c >>= 1)
        if (V % c == 0 && (al & (c * sizeof(IO) - 1)) == 0) { vec = c; break; }
    const int64_t total = cells * (int64_t)V / vec;
    const Problem p = lay ? *lay : Problem{};
    // compact: CTAs per lattice from the rows a CTA covers in kCompactIters iterations (rounded up to whole rows)
    const dim3 grid = lay ? dim3(compact_gx(STU, N, ((int64_t)kLogitThreads * vec * kCompactIters + V - 1) / V), N)
                          : dim3((unsigned)min((total + kLogitThreads - 1) / kLogitThreads, (int64_t)sms * 32));
    const int64_t stride = (int64_t)grid.x * kLogitThreads * vec;
    const int64_t srows = stride / V;
    const int sv = (int)(stride - srows * V);
#define RNNT_EXPAND_LAUNCH(VEC)                                                                                            \
    (hat ? (lay ? k_expand_logits_hat<IO, VEC, kRowsCompact><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, ranges, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv, p) \
            : ranges ? k_expand_logits_hat<IO, VEC, kRowsPruned><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, ranges, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv, p) \
                : k_expand_logits_hat<IO, VEC, kRowsDense><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, ranges, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv, p)) \
     : lay ? k_expand_logits<IO, VEC, true><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv, p) \
     : ranges ? k_expand_logits_pruned<IO, VEC><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, ranges, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv) \
         : k_expand_logits<IO, VEC><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv, p))
    if constexpr (sizeof(IO) == 2) {
        if (vec == 8) RNNT_EXPAND_LAUNCH(8);
        else if (vec == 4) RNNT_EXPAND_LAUNCH(4);
        else if (vec == 2) RNNT_EXPAND_LAUNCH(2);
        else RNNT_EXPAND_LAUNCH(1);
    } else {
        if (vec == 4) RNNT_EXPAND_LAUNCH(4);
        else if (vec == 2) RNNT_EXPAND_LAUNCH(2);
        else RNNT_EXPAND_LAUNCH(1);
    }
#undef RNNT_EXPAND_LAUNCH
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_expand_logits(cudaStream_t s, const void *x, const float *lse, const float2 *pg, const int *labels,
                                 const float *grad_out, void *out, int N, int T, int U, int V, int blank, int io_bf16,
                                 int hat) {
    if (io_bf16)
        return expand_logits_as(s, static_cast<const __nv_bfloat16 *>(x), lse, pg, labels, grad_out,
                                static_cast<__nv_bfloat16 *>(out), N, T, U, V, blank, nullptr, 0, nullptr, 0, hat);
    return expand_logits_as(s, static_cast<const float *>(x), lse, pg, labels, grad_out, static_cast<float *>(out), N, T,
                            U, V, blank, nullptr, 0, nullptr, 0, hat);
}

cudaError_t launch_expand_logits_compact(cudaStream_t s, const void *x, const float *lse, const float2 *pg,
                                         const Problem &p, const int *labels, const float *grad_out, void *out,
                                         int64_t STU, int V, int blank, int io_bf16, int hat) {
    if (io_bf16)
        return expand_logits_as(s, static_cast<const __nv_bfloat16 *>(x), lse, pg, labels, grad_out,
                                static_cast<__nv_bfloat16 *>(out), p.N, 0, 0, V, blank, &p, STU, nullptr, 0, hat);
    return expand_logits_as(s, static_cast<const float *>(x), lse, pg, labels, grad_out, static_cast<float *>(out), p.N,
                            0, 0, V, blank, &p, STU, nullptr, 0, hat);
}

cudaError_t launch_lse_pairs_pruned(cudaStream_t s, const void *x, const int *labels, const int *ranges, int N, int T,
                                    int S, int U, int V, int blank, float2 *pairs, float *lse, int io_bf16, int hat) {
    if (io_bf16)
        return lse_pairs_as(s, static_cast<const __nv_bfloat16 *>(x), labels, N, T, U, V, blank, pairs, lse, nullptr, 0,
                            ranges, S, hat);
    return lse_pairs_as(s, static_cast<const float *>(x), labels, N, T, U, V, blank, pairs, lse, nullptr, 0, ranges, S,
                        hat);
}

cudaError_t launch_expand_logits_pruned(cudaStream_t s, const void *x, const float *lse, const float2 *pg,
                                        const int *labels, const int *ranges, const float *grad_out, void *out, int N,
                                        int T, int S, int U, int V, int blank, int io_bf16, int hat) {
    if (io_bf16)
        return expand_logits_as(s, static_cast<const __nv_bfloat16 *>(x), lse, pg, labels, grad_out,
                                static_cast<__nv_bfloat16 *>(out), N, T, U, V, blank, nullptr, 0, ranges, S, hat);
    return expand_logits_as(s, static_cast<const float *>(x), lse, pg, labels, grad_out, static_cast<float *>(out), N, T,
                            U, V, blank, nullptr, 0, ranges, S, hat);
}

}  // namespace rnnt
