// simple.cu -- the "simple" transducer loss of the pruned recipe (k2's rnnt_loss_simple, regular lattice) and the
// prune ranges chosen from its occupation probabilities (k2's get_rnnt_prune_ranges + _adjust_pruning_lower_bound).
//
// The simple joint of lattice n is am[n,t,:] + lm[n,u,:] with am (N,T,V) and lm (N,U,V).  Its normaliser factorises:
// with offsets oa[t] = max_v am[t,v], ol[u] = max_v lm[u,v] (0 for a row whose maximum is -inf),
// Ea[t,v] = exp(am[t,v] - oa[t]) and El[u,v] = exp(lm[u,v] - ol[u]),
//
//   Z[t,u]    = sum_v Ea[t,v] El[u,v]                       a (T,V) x (V,U) product per lattice
//   norm[t,u] = log(max(Z, FLT_MIN)) + oa[t] + ol[u]
//
// so no (N,T,U,V) tensor is formed.  Kernels:
//
//   k_row_offsets    oa (N,T) and ol (N,U), one warp per row
//   k_simple_mm      a tiled fp32 FFMA contraction (no tensor cores: TF32 would put ~1e-3 on every log-prob) with
//                    the exponentials taken as tiles are loaded.  Three modes:
//                      kMmNorm  Z over K = V; the epilogue writes norm and the (blank, label) pairs of every cell
//                      kMmDam   sum_u W[t,u] El[u,v] over K = U; the epilogue writes -(Ea * it) into dam
//                      kMmDlm   sum_t W[t,u] Ea[t,v] over K = T; the epilogue writes -(El * it) into dlm
//                    with W[t,u] = grad_out[n] (gb + gl)[t,u] / Z[t,u] from the (N,T,U,2) pair gradients.
//   k_simple_sparse  adds the (blank, label) terms of the gradients: one thread per row, a fixed loop order, no atomics
//   k_prune_ranges   one CTA per lattice: each frame's best window start, then the two suffix-minimum passes
//
// Rows and columns past a lattice's lengths are never read (a NaN in padding stays out of every sum); their outputs are
// written as 0.  A lattice with invalid lengths has no cells at all.
#include <cfloat>
#include <climits>

#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kMmThreads = 256, kBM = 64, kBN = 64, kBK = 16;
constexpr int kRowThreads = 256;
constexpr int kRangeThreads = 1024;            // k_prune_ranges: 32 warps, one frame each, per lattice

// lattice n's (Tn, Un), or (0, 0) when xn outside [1, T] or yn + 1 outside [1, U]
__device__ __forceinline__ void simple_lengths(const int *xn, const int *yn, int n, int T, int U, int &Tn, int &Un) {
    const int a = xn[n], b = yn[n];
    const bool ok = a >= 1 && a <= T && b >= 0 && b < U;
    Tn = ok ? a : 0;
    Un = ok ? b + 1 : 0;
}

// rows [0, rows_a) are am's (N*T), [rows_a, rows) lm's (N*U); one warp per row
__global__ void __launch_bounds__(kRowThreads)
k_row_offsets(const float *__restrict__ am, const float *__restrict__ lm, int64_t rows_a, int64_t rows, int V,
              float *__restrict__ off_a, float *__restrict__ off_l) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * kRowThreads + threadIdx.x) >> 5; r < rows;
         r += (int64_t)gridDim.x * (kRowThreads / 32)) {
        const bool is_a = r < rows_a;
        const float *x = is_a ? am + r * V : lm + (r - rows_a) * V;
        float m = -INFINITY;
        for (int v = lane; v < V; v += 32) m = fmaxf(m, __ldg(x + v));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        // a row of -inf only: offset 0, so that its exponentials are exp(-inf) = 0 rather than exp(-inf + inf) = NaN
        if (lane == 0) (is_a ? off_a[r] : off_l[r - rows_a]) = (m == -INFINITY) ? 0.0f : m;
    }
}

enum { kMmNorm = 0, kMmDam = 1, kMmDlm = 2 };

// W[t,u] = grad_out[n] (gb + gl) / Z, with 1/Z = exp(oa + ol - norm)
__device__ __forceinline__ float simple_w(const SimpleArgs &a, int64_t nt, int n, int t, int u, float g) {
    const float2 q = a.pg[nt * a.U + u];
    return (g * (q.x + q.y)) * expf((a.off_a[(int64_t)n * a.T + t] + a.off_l[(int64_t)n * a.U + u]) - a.norm[nt * a.U + u]);
}

// One 64 x 64 output tile of lattice blockIdx.z: rows m (t, t, u), columns c (u, v, v), reduction k (v, u, t) for
// MODE kMmNorm, kMmDam, kMmDlm.  256 threads, 4 x 4 outputs each; every output is summed over k in increasing order.
template <int MODE>
__global__ void __launch_bounds__(kMmThreads) k_simple_mm(SimpleArgs a) {
    __shared__ __align__(16) float As[kBK][kBM];
    __shared__ __align__(16) float Bs[kBK][kBN];
    const int n = blockIdx.z, T = a.T, U = a.U, V = a.V;
    int Tn, Un;
    simple_lengths(a.xn, a.yn, n, T, U, Tn, Un);
    const int Mlim = MODE == kMmDlm ? Un : Tn;                 // live rows, columns, reduction length
    const int Clim = MODE == kMmNorm ? Un : V;
    const int Klim = MODE == kMmNorm ? V : MODE == kMmDam ? Un : Tn;
    const int m0 = blockIdx.y * kBM, c0 = blockIdx.x * kBN;
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const float g = (MODE != kMmNorm && a.grad_out) ? a.grad_out[n] : 1.0f;
    const float *am = a.am + (int64_t)n * T * V, *lm = a.lm + (int64_t)n * U * V;
    const float *oa = a.off_a + (int64_t)n * T, *ol = a.off_l + (int64_t)n * U;
    const int64_t nT = (int64_t)n * T;
    float acc[4][4] = {};
    if (m0 < Mlim && c0 < Clim) {
        for (int k0 = 0; k0 < Klim; k0 += kBK) {
            // A tile As[k][m]: for kMmNorm / kMmDam the source is contiguous along k (thread: row tid / 4, 4 k's),
            // for kMmDlm along m (thread: k = tid / 16, 4 m's)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if constexpr (MODE == kMmDlm) {
                    const int kk = tid / 16, mm = (tid % 16) * 4 + j, t = k0 + kk, u = m0 + mm;
                    As[kk][mm] = (t < Tn && u < Un) ? simple_w(a, nT + t, n, t, u, g) : 0.0f;
                } else {
                    const int mm = tid / 4, kk = (tid % 4) * 4 + j, t = m0 + mm, k = k0 + kk;
                    float v = 0.0f;
                    if (MODE == kMmNorm && t < Tn && k < V) v = expf(__ldg(am + (int64_t)t * V + k) - oa[t]);
                    if (MODE == kMmDam && t < Tn && k < Un) v = simple_w(a, nT + t, n, t, k, g);
                    As[kk][mm] = v;
                }
            }
            // B tile Bs[k][c]: kMmNorm's source (lm rows) is contiguous along k, the others' along c
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if constexpr (MODE == kMmNorm) {
                    const int cc = tid / 4, kk = (tid % 4) * 4 + j, u = c0 + cc, k = k0 + kk;
                    Bs[kk][cc] = (u < Un && k < V) ? expf(__ldg(lm + (int64_t)u * V + k) - ol[u]) : 0.0f;
                } else {
                    const int kk = tid / 16, cc = (tid % 16) * 4 + j, r = k0 + kk, v = c0 + cc;
                    float e = 0.0f;
                    if (MODE == kMmDam && r < Un && v < V) e = expf(__ldg(lm + (int64_t)r * V + v) - ol[r]);
                    if (MODE == kMmDlm && r < Tn && v < V) e = expf(__ldg(am + (int64_t)r * V + v) - oa[r]);
                    Bs[kk][cc] = e;
                }
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < kBK; ++k) {
                const float4 x = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
                const float4 y = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
                const float xa[4] = {x.x, x.y, x.z, x.w}, yb[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(xa[i], yb[jj], acc[i][jj]);
            }
            __syncthreads();
        }
    }
    // epilogue: every in-bounds output of the tile is written, 0 outside the lattice
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int c = c0 + tx * 4 + jj;
            if constexpr (MODE == kMmNorm) {
                if (m >= T || c >= U) continue;
                const int64_t cell = (nT + m) * U + c;
                float nm = 0.0f;
                float2 pr = make_float2(0.0f, 0.0f);
                if (m < Tn && c < Un) {
                    const float z = acc[i][jj] < FLT_MIN ? FLT_MIN : acc[i][jj];     // (NaN stays NaN)
                    nm = (logf(z) + oa[m]) + ol[c];
                    const int y = (c < Un - 1) ? a.labels[(int64_t)n * (U - 1) + c] : a.blank;
                    const float *ra = am + (int64_t)m * V, *rl = lm + (int64_t)c * V;
                    pr = make_float2((__ldg(ra + a.blank) + __ldg(rl + a.blank)) - nm, (__ldg(ra + y) + __ldg(rl + y)) - nm);
                }
                a.norm[cell] = nm;
                a.pairs[cell] = pr;
            } else {
                const int rows = MODE == kMmDam ? T : U;
                if (m >= rows || c >= V) continue;
                float r = 0.0f;
                if (m < Mlim) {
                    const float e = MODE == kMmDam ? expf(__ldg(am + (int64_t)m * V + c) - oa[m])
                                                   : expf(__ldg(lm + (int64_t)m * V + c) - ol[m]);
                    r = -(e * acc[i][jj]);
                }
                a.out[((int64_t)n * rows + m) * V + c] = r;
            }
        }
    }
}

// The (blank, label) terms of the gradients, added to what k_simple_mm wrote: thread r < N*T owns dam row (n,t) and
// adds grad_out * gl[t,u] at v = labels[u] for u = 0 .. Un-2 in turn, then grad_out * sum_u gb[t,u] at blank; thread
// r >= N*T owns dlm row (n,u) and adds grad_out * sum_t gb[t,u] at blank, then grad_out * sum_t gl[t,u] at labels[u].
// Sums run in increasing index; a label equal to blank receives both terms.
__global__ void __launch_bounds__(kRowThreads) k_simple_sparse(SimpleArgs a, float *__restrict__ dam, float *__restrict__ dlm, int N) {
    const int T = a.T, U = a.U, V = a.V;
    const int64_t rows_a = (int64_t)N * T, rows = rows_a + (int64_t)N * U;
    for (int64_t r = (int64_t)blockIdx.x * kRowThreads + threadIdx.x; r < rows; r += (int64_t)gridDim.x * kRowThreads) {
        const bool is_a = r < rows_a;
        const int n = (int)(is_a ? r / T : (r - rows_a) / U);
        const int i = (int)(is_a ? r % T : (r - rows_a) % U);
        int Tn, Un;
        simple_lengths(a.xn, a.yn, n, T, U, Tn, Un);
        const float g = a.grad_out ? a.grad_out[n] : 1.0f;
        const int *lab = a.labels + (int64_t)n * (U - 1);
        if (is_a) {
            if (i >= Tn) continue;
            const float2 *q = a.pg + r * U;
            float *o = dam + r * V;
            float sb = 0.0f;
            for (int u = 0; u < Un; ++u) {
                const float2 p = q[u];
                sb += p.x;
                if (u < Un - 1) o[lab[u]] += g * p.y;
            }
            o[a.blank] += g * sb;
        } else {
            if (i >= Un) continue;
            const float2 *q = a.pg + (int64_t)n * T * U + i;
            float *o = dlm + (r - rows_a) * V;
            float sb = 0.0f, sl = 0.0f;
            for (int t = 0; t < Tn; ++t) {
                const float2 p = q[(int64_t)t * U];
                sb += p.x;
                sl += p.y;
            }
            o[a.blank] += g * sb;
            if (i < Un - 1) o[lab[i]] += g * sl;
        }
    }
}

// One CTA per lattice.  Frame t < Tn-1 takes the first r in [0, Un-S] with the largest
// score(t,r) = (ob[t,r] + ... + ob[t,r+S-1]) - (r > 0 ? ol[t,r-1] : 0), ob = -gb, ol = -gl, the sum added in increasing
// u and the subtraction last; a NaN score never wins, and r = 0 when every score is NaN.  Frames t >= Tn-1 take Un-S.
// One warp per frame, lane l scoring r = l, l+32, ...  Then, over all T frames: b = suffix minimum of r0,
// c = k t - b, c' = suffix minimum of c, r = k t - max(c', 0) -- computed in place in `ranges` by warp 0.  TYPE is the
// lattice type: k = S-1 for 0 (regular), 1 for 1 and 2 (modified, constrained); type 2 takes gb from raw (the blank
// slots before the constrained fold), the others from pg.
template <int TYPE>
__global__ void __launch_bounds__(kRangeThreads)
k_prune_ranges(const float2 *__restrict__ pg, const int *__restrict__ xn, const int *__restrict__ yn, int T, int U,
               int S, int *__restrict__ ranges, const float *__restrict__ raw) {
    const int n = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int Tn, Un;
    simple_lengths(xn, yn, n, T, U, Tn, Un);
    int *out = ranges + (int64_t)n * T;
    if (Tn == 0 || Un <= S) {
        for (int t = threadIdx.x; t < T; t += kRangeThreads) out[t] = 0;
        return;
    }
    const int top = Un - S;
    for (int t = warp; t < T; t += kRangeThreads / 32) {
        int best_r = top;
        if (t < Tn - 1) {
            const float2 *q = pg + ((int64_t)n * T + t) * U;
            bool have = false;
            float best = 0.0f;
            best_r = 0;
            for (int r = lane; r <= top; r += 32) {
                float sc = 0.0f;
                if constexpr (TYPE == 2) {
                    const float *qb = raw + ((int64_t)n * T + t) * U;
                    for (int u = r; u < r + S; ++u) sc += -qb[u];
                } else {
                    for (int u = r; u < r + S; ++u) sc += -q[u].x;
                }
                if (r > 0) sc = sc - (-q[r - 1].y);
                if (sc == sc && (!have || sc > best)) { best = sc; best_r = r; have = true; }
            }
            // first r of the largest score across the lanes: a lane without a number loses, ties go to the smaller r
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const int h2 = __shfl_xor_sync(0xffffffffu, (int)have, o), r2 = __shfl_xor_sync(0xffffffffu, best_r, o);
                const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
                const bool take = h2 && (!have || b2 > best || (b2 == best && r2 < best_r));
                if (take) { best = b2; best_r = r2; have = true; }
            }
            if (!have) best_r = 0;
        }
        if (lane == 0) out[t] = best_r;
    }
    __syncthreads();
    if (warp != 0) return;
    int carry_b = INT_MAX, carry_c = INT_MAX;
    for (int base = ((T - 1) / 32) * 32; base >= 0; base -= 32) {
        const int t = base + lane;
        int b = t < T ? out[t] : INT_MAX;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_down_sync(0xffffffffu, b, o);
            if (lane + o < 32) b = min(b, y);
        }
        b = min(b, carry_b);
        carry_b = __shfl_sync(0xffffffffu, b, 0);
        int c = t < T ? (TYPE == 0 ? S - 1 : 1) * t - b : INT_MAX;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_down_sync(0xffffffffu, c, o);
            if (lane + o < 32) c = min(c, y);
        }
        c = min(c, carry_c);
        carry_c = __shfl_sync(0xffffffffu, c, 0);
        if (t < T) out[t] = (TYPE == 0 ? S - 1 : 1) * t - max(c, 0);
    }
}

static int row_grid(int64_t rows, int per_cta) {
    return (int)max((int64_t)1, min((rows + per_cta - 1) / per_cta, (int64_t)sm_count(current_device()) * 16));
}

cudaError_t launch_simple_forward(cudaStream_t s, const SimpleArgs &a, int N) {
    const int64_t rows_a = (int64_t)N * a.T, rows = rows_a + (int64_t)N * a.U;
    k_row_offsets<<<row_grid(rows, kRowThreads / 32), kRowThreads, 0, s>>>(a.am, a.lm, rows_a, rows, a.V, a.off_a,
                                                                            a.off_l);
    count_launch();
    const dim3 grid((a.U + kBN - 1) / kBN, (a.T + kBM - 1) / kBM, N);
    k_simple_mm<kMmNorm><<<grid, kMmThreads, 0, s>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_simple_backward(cudaStream_t s, const SimpleArgs &a, float *dam, float *dlm, int N) {
    SimpleArgs b = a;
    b.out = dam;
    k_simple_mm<kMmDam><<<dim3((a.V + kBN - 1) / kBN, (a.T + kBM - 1) / kBM, N), kMmThreads, 0, s>>>(b);
    count_launch();
    b.out = dlm;
    k_simple_mm<kMmDlm><<<dim3((a.V + kBN - 1) / kBN, (a.U + kBM - 1) / kBM, N), kMmThreads, 0, s>>>(b);
    count_launch();
    const int64_t rows = (int64_t)N * (a.T + a.U);
    k_simple_sparse<<<row_grid(rows, kRowThreads), kRowThreads, 0, s>>>(a, dam, dlm, N);
    count_launch();
    return cudaGetLastError();
}

// ---- k2's smoothed simple loss (rnnt_loss_smoothed: lm_only_scale sl, am_only_scale sa, c = 1 - sl - sa) ----------
//
//   Ll[n,u] = log(sum_v exp(lm[u,v] - ol[u])) + ol[u]          p[n,u,v] = exp(lm[u,v] - Ll[u])
//   uni[v]  = (sum over every lm row of p[.,v]) / (N U) + FLT_MIN
//   Am[n,t] = log(sum_v exp(am[t,v] - oa[t]) uni[v]) + oa[t]
//   pair_k  = (c simple_k + sl (lm[u,k] - Ll[u])) + sa ((am[t,k] + log uni[k]) - Am[t]),   a zero-scale term absent
//
//   k_smooth_lm_rows     Ll, one warp per row; with sa > 0 also the unigram partial of its CTA's kSmoothRows rows
//   k_smooth_uni         uni and log uni: one thread per v sums the partials in CTA order
//   k_smooth_am_norm     Am, one warp per row
//   k_smooth_mix         the mixed pairs, one thread per cell, in place
//   k_smooth_cols        backward: Cb[n,u] = sum_t gb, Cl[n,u] = sum_t gl (one thread per column), and c*grad_out
//   k_smooth_am_rows     the sa terms of dam, and the partials of G's dense part, kSmoothRows am rows per CTA
//   k_smooth_G           G[v] = sa (Gs[v] / uni[v] - Gd[v]); Gs is the blank / label scatter, found by a scan
//   k_smooth_lm_rows_bwd the sl and unigram terms of dlm, one warp per row
//
// Every reduction is partitioned by the shapes alone (fixed rows per CTA, warp-strided rows, fixed loop orders), so
// the bits do not depend on the grid size or the SM count; there are no atomics.

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// CTA b owns lm rows [b kSmoothRows, (b+1) kSmoothRows) of the flattened (N*U); 8 warps, 4 rows each.  With sa = 0 only
// live rows (u < Un) are read, and the others get Ll = 0.
__global__ void __launch_bounds__(kRowThreads) k_smooth_lm_rows(SmoothArgs m) {
    __shared__ float Ls[kSmoothRows];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t rows = (int64_t)m.N * m.U, r0 = (int64_t)blockIdx.x * kSmoothRows;
    const int V = m.V;
    for (int i = warp; i < kSmoothRows; i += kRowThreads / 32) {
        const int64_t r = r0 + i;
        if (r >= rows) break;
        const int n = (int)(r / m.U), u = (int)(r % m.U);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, m.T, m.U, Tn, Un);
        float L = 0.0f;
        if (m.sa > 0.0f || u < Un) {
            const float *x = m.lm + r * V, o = m.off_l[r];
            float s = 0.0f;
            for (int v = lane; v < V; v += 32) s += expf(__ldg(x + v) - o);
            L = logf(warp_sum(s)) + o;
        }
        if (lane == 0) { m.Ll[r] = L; Ls[i] = L; }
    }
    if (!(m.sa > 0.0f)) return;
    __syncthreads();
    const int nr = (int)min((int64_t)kSmoothRows, rows - r0);
    for (int v = threadIdx.x; v < V; v += kRowThreads) {
        float acc = 0.0f;
        for (int i = 0; i < nr; ++i) acc += expf(__ldg(m.lm + (r0 + i) * V + v) - Ls[i]);
        m.upart[(int64_t)blockIdx.x * V + v] = acc;
    }
}

__global__ void __launch_bounds__(kRowThreads) k_smooth_uni(SmoothArgs m, int parts) {
    const int v = blockIdx.x * kRowThreads + threadIdx.x;
    if (v >= m.V) return;
    float s = 0.0f;
    for (int b = 0; b < parts; ++b) s += m.upart[(int64_t)b * m.V + v];
    const float u = __fadd_rn(__fdiv_rn(s, (float)((int64_t)m.N * m.U)), FLT_MIN);
    m.uni[v] = u;
    m.loguni[v] = logf(u);
}

// one warp per am row; rows past Tn (and every row of a lattice with invalid lengths) get Am = 0 and are not read
__global__ void __launch_bounds__(kRowThreads) k_smooth_am_norm(SmoothArgs m) {
    const int lane = threadIdx.x & 31;
    const int64_t rows = (int64_t)m.N * m.T;
    for (int64_t r = ((int64_t)blockIdx.x * kRowThreads + threadIdx.x) >> 5; r < rows;
         r += (int64_t)gridDim.x * (kRowThreads / 32)) {
        const int n = (int)(r / m.T), t = (int)(r % m.T);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, m.T, m.U, Tn, Un);
        float A = 0.0f;
        if (t < Tn) {
            const float *x = m.am + r * m.V, o = m.off_a[r];
            float s = 0.0f;
            for (int v = lane; v < m.V; v += 32) s = fmaf(expf(__ldg(x + v) - o), m.uni[v], s);
            A = logf(warp_sum(s)) + o;
        }
        if (lane == 0) m.Am[r] = A;
    }
}

// pair_k = (c simple_k + sl lmonly_k) + sa amonly_k in round-to-nearest steps (no contraction), each term only when its
// scale is not 0; cells outside the lattice keep (0, 0)
__device__ __forceinline__ float smooth_pair(const SmoothArgs &m, float simple, const float *ra, const float *rl,
                                             float Ll, float Am, int k) {
    float p = __fmul_rn(m.c, simple);
    if (m.sl > 0.0f) p = __fadd_rn(p, __fmul_rn(m.sl, __fsub_rn(__ldg(rl + k), Ll)));
    if (m.sa > 0.0f) p = __fadd_rn(p, __fmul_rn(m.sa, __fsub_rn(__fadd_rn(__ldg(ra + k), m.loguni[k]), Am)));
    return p;
}

__global__ void __launch_bounds__(kRowThreads) k_smooth_mix(SmoothArgs m) {
    const int T = m.T, U = m.U, V = m.V;
    const int64_t cells = (int64_t)m.N * T * U;
    for (int64_t i = (int64_t)blockIdx.x * kRowThreads + threadIdx.x; i < cells; i += (int64_t)gridDim.x * kRowThreads) {
        const int u = (int)(i % U);
        const int64_t nt = i / U;
        const int t = (int)(nt % T), n = (int)(nt / T);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, T, U, Tn, Un);
        if (t >= Tn || u >= Un) continue;
        const int y = (u < Un - 1) ? m.labels[(int64_t)n * (U - 1) + u] : m.blank;
        const float *ra = m.am + nt * V, *rl = m.lm + ((int64_t)n * U + u) * V;
        const float Ll = m.sl > 0.0f ? m.Ll[(int64_t)n * U + u] : 0.0f, Am = m.sa > 0.0f ? m.Am[nt] : 0.0f;
        const float2 q = m.pairs[i];
        m.pairs[i] = make_float2(smooth_pair(m, q.x, ra, rl, Ll, Am, m.blank), smooth_pair(m, q.y, ra, rl, Ll, Am, y));
    }
}

// thread r < N*U owns column (n,u): Cb, Cl summed over t < Tn in increasing t (0 outside the lattice); thread r < N
// also writes cgo[r] = c * grad_out[r]
__global__ void __launch_bounds__(kRowThreads) k_smooth_cols(SmoothArgs m) {
    const int T = m.T, U = m.U;
    const int64_t rows = (int64_t)m.N * U;
    for (int64_t r = (int64_t)blockIdx.x * kRowThreads + threadIdx.x; r < rows; r += (int64_t)gridDim.x * kRowThreads) {
        const int n = (int)(r / U), u = (int)(r % U);
        if (r < m.N) m.cgo[r] = __fmul_rn(m.c, m.grad_out ? m.grad_out[r] : 1.0f);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, T, U, Tn, Un);
        float sb = 0.0f, sl = 0.0f;
        if (u < Un) {
            const float2 *q = m.pg + (int64_t)n * T * U + u;
            for (int t = 0; t < Tn; ++t) {
                const float2 p = q[(int64_t)t * U];
                sb += p.x;
                sl += p.y;
            }
        }
        m.cb[r] = sb;
        m.cl[r] = sl;
    }
}

// CTA b owns am rows [b kSmoothRows, (b+1) kSmoothRows) of the flattened (N*T).  Per live row (t < Tn), with
// go = grad_out[n], Ra = sum_u (gb + gl), Sb = sum_u gb (one warp, lane-strided u, then a butterfly):
//   dam[t,v] += -(sa go Ra) (exp(am[t,v] - Am[t]) uni[v])                     (thread per v, rows in order)
//   gpart[b,v] = sum over the CTA's live rows of (go Ra) exp(am[t,v] - Am[t])  (the same loop)
//   then dam[t,y_u] += sa go gl[t,u] for u < Un-1 in turn, dam[t,blank] += sa go Sb   (thread per row)
// uni[v] is taken as expf(log uni[v]).
__global__ void __launch_bounds__(kRowThreads) k_smooth_am_rows(SmoothArgs m, float *__restrict__ dam) {
    __shared__ float As[kSmoothRows], Ws[kSmoothRows], Qs[kSmoothRows], Bs[kSmoothRows];
    __shared__ bool Live[kSmoothRows];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int T = m.T, U = m.U, V = m.V;
    const int64_t rows = (int64_t)m.N * T, r0 = (int64_t)blockIdx.x * kSmoothRows;
    const int nr = (int)min((int64_t)kSmoothRows, rows - r0);
    for (int i = warp; i < nr; i += kRowThreads / 32) {
        const int64_t r = r0 + i;
        const int n = (int)(r / T), t = (int)(r % T);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, T, U, Tn, Un);
        float ra = 0.0f, sb = 0.0f, go = 0.0f;
        const bool live = t < Tn;
        if (live) {
            go = m.grad_out ? m.grad_out[n] : 1.0f;
            const float2 *q = m.pg + r * U;
            for (int u = lane; u < Un; u += 32) {
                const float2 p = q[u];
                ra += p.x + p.y;
                sb += p.x;
            }
            ra = warp_sum(ra);
            sb = warp_sum(sb);
        }
        if (lane == 0) {
            Live[i] = live;
            As[i] = m.Am[r];
            Ws[i] = -(m.sa * go * ra);
            Qs[i] = go * ra;
            Bs[i] = __fmul_rn(m.sa, go) * sb;
        }
    }
    __syncthreads();
    for (int v = threadIdx.x; v < V; v += kRowThreads) {
        const float un = expf(m.loguni[v]);
        float acc = 0.0f;
        for (int i = 0; i < nr; ++i) {
            if (!Live[i]) continue;
            const int64_t r = r0 + i;
            const float e = expf(__ldg(m.am + r * V + v) - As[i]);
            dam[r * V + v] = __fadd_rn(dam[r * V + v], __fmul_rn(Ws[i], __fmul_rn(e, un)));
            acc = __fadd_rn(acc, __fmul_rn(Qs[i], e));
        }
        m.gpart[(int64_t)blockIdx.x * V + v] = acc;
    }
    __syncthreads();
    if (threadIdx.x < nr) {
        const int i = threadIdx.x;
        const int64_t r = r0 + i;
        const int n = (int)(r / T);
        if (Live[i]) {
            const int Un = m.yn[n] + 1;                // live rows belong to lattices with valid lengths
            const float w = __fmul_rn(m.sa, m.grad_out ? m.grad_out[n] : 1.0f);
            const float2 *q = m.pg + r * U;
            const int *lab = m.labels + (int64_t)n * (U - 1);
            float *o = dam + r * V;
            for (int u = 0; u < Un - 1; ++u) o[lab[u]] += w * q[u].y;
            o[m.blank] += Bs[i];
        }
    }
}

// One thread per v (CTAs of kRowThreads over V).  Gd[v] = the gpart column summed in CTA order.  Gs[v] = sum over the
// flattened (n,u) in order of go_n Cb[n,u] when v = blank (u < Un) and go_n Cl[n,u] when v = labels[n,u] (u < Un-1),
// the blank term of an entry before its label term: every CTA stages kRowThreads entries in shared memory at a time
// and each thread scans them for its v.
__global__ void __launch_bounds__(kRowThreads) k_smooth_G(SmoothArgs m, int parts) {
    __shared__ int Yb[kRowThreads], Yl[kRowThreads];
    __shared__ float Fb[kRowThreads], Fl[kRowThreads];
    const int v = blockIdx.x * kRowThreads + threadIdx.x, U = m.U;
    const int64_t ents = (int64_t)m.N * U;
    float gs = 0.0f;
    for (int64_t j0 = 0; j0 < ents; j0 += kRowThreads) {
        const int64_t j = j0 + threadIdx.x;
        int yb = -1, yl = -1;
        float fb = 0.0f, fl = 0.0f;
        if (j < ents) {
            const int n = (int)(j / U), u = (int)(j % U);
            int Tn, Un;
            simple_lengths(m.xn, m.yn, n, m.T, U, Tn, Un);
            if (u < Un) {
                const float go = m.grad_out ? m.grad_out[n] : 1.0f;
                yb = m.blank;
                fb = go * m.cb[j];
                if (u < Un - 1) { yl = m.labels[(int64_t)n * (U - 1) + u]; fl = go * m.cl[j]; }
            }
        }
        Yb[threadIdx.x] = yb; Yl[threadIdx.x] = yl; Fb[threadIdx.x] = fb; Fl[threadIdx.x] = fl;
        __syncthreads();
        const int k1 = (int)min((int64_t)kRowThreads, ents - j0);
        for (int k = 0; k < k1; ++k) {
            if (Yb[k] == v) gs += Fb[k];
            if (Yl[k] == v) gs += Fl[k];
        }
        __syncthreads();
    }
    if (v >= m.V) return;
    float gd = 0.0f;
    for (int b = 0; b < parts; ++b) gd += m.gpart[(int64_t)b * m.V + v];
    m.G[v] = __fmul_rn(m.sa, __fsub_rn(__fdiv_rn(gs, expf(m.loguni[v])), gd));
}

// One warp per lm row (n,u).  With p[v] = exp(lm[u,v] - Ll[u]) and, when sa > 0, pG = sum_v p[v] G[v] (lane-strided,
// then a butterfly):
//   dlm[u,v] += -(sl go (Cb + Cl)[u]) p[v]           (sl > 0, live rows u < Un)
//   dlm[u,v] += (p[v] (G[v] - pG)) / (N U)           (sa > 0, every row)
//   then dlm[u,blank] += sl go Cb[u], dlm[u,y_u] += sl go Cl[u] for u < Un-1   (sl > 0, live rows; lane 0)
// With sa = 0 rows past Un are not read.
__global__ void __launch_bounds__(kRowThreads) k_smooth_lm_rows_bwd(SmoothArgs m, float *__restrict__ dlm) {
    const int lane = threadIdx.x & 31;
    const int U = m.U, V = m.V;
    const int64_t rows = (int64_t)m.N * U;
    const bool sa = m.sa > 0.0f, sl = m.sl > 0.0f;
    const float nu = (float)rows;
    for (int64_t r = ((int64_t)blockIdx.x * kRowThreads + threadIdx.x) >> 5; r < rows;
         r += (int64_t)gridDim.x * (kRowThreads / 32)) {
        const int n = (int)(r / U), u = (int)(r % U);
        int Tn, Un;
        simple_lengths(m.xn, m.yn, n, m.T, U, Tn, Un);
        const bool live = sl && u < Un;
        if (!sa && !live) continue;
        const float *x = m.lm + r * V, L = m.Ll[r];
        float *o = dlm + r * V;
        float pG = 0.0f;
        if (sa) {
            for (int v = lane; v < V; v += 32) pG = fmaf(expf(__ldg(x + v) - L), m.G[v], pG);
            pG = warp_sum(pG);
        }
        const float go = m.grad_out ? m.grad_out[n] : 1.0f;
        const float wl = live ? -(m.sl * go * (m.cb[r] + m.cl[r])) : 0.0f;
        for (int v = lane; v < V; v += 32) {
            const float p = expf(__ldg(x + v) - L);
            float d = o[v];
            if (live) d = __fadd_rn(d, __fmul_rn(wl, p));
            if (sa) d = __fadd_rn(d, __fdiv_rn(__fmul_rn(p, __fsub_rn(m.G[v], pG)), nu));
            o[v] = d;
        }
        if (live) {
            __syncwarp();
            if (lane == 0) {
                const float w = __fmul_rn(m.sl, go);
                o[m.blank] += w * m.cb[r];
                if (u < Un - 1) o[m.labels[(int64_t)n * (U - 1) + u]] += w * m.cl[r];
            }
            __syncwarp();
        }
    }
}

cudaError_t launch_simple_smoothed_forward(cudaStream_t s, const SmoothArgs &m) {
    const int64_t lrows = (int64_t)m.N * m.U, arows = (int64_t)m.N * m.T;
    const int lparts = (int)((lrows + kSmoothRows - 1) / kSmoothRows);
    k_smooth_lm_rows<<<lparts, kRowThreads, 0, s>>>(m);
    count_launch();
    if (m.sa > 0.0f) {
        k_smooth_uni<<<(m.V + kRowThreads - 1) / kRowThreads, kRowThreads, 0, s>>>(m, lparts);
        count_launch();
        k_smooth_am_norm<<<row_grid(arows, kRowThreads / 32), kRowThreads, 0, s>>>(m);
        count_launch();
    }
    k_smooth_mix<<<row_grid((int64_t)m.N * m.T * m.U, kRowThreads), kRowThreads, 0, s>>>(m);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_simple_smoothed_backward(cudaStream_t s, const SimpleArgs &a, const SmoothArgs &m, float *dam,
                                            float *dlm) {
    const int64_t lrows = (int64_t)m.N * m.U, arows = (int64_t)m.N * m.T;
    k_smooth_cols<<<row_grid(lrows, kRowThreads), kRowThreads, 0, s>>>(m);
    count_launch();
    SimpleArgs b = a;
    b.grad_out = m.cgo;
    cudaError_t e = launch_simple_backward(s, b, dam, dlm, m.N);
    if (e != cudaSuccess) return e;
    if (m.sa > 0.0f) {
        const int aparts = (int)((arows + kSmoothRows - 1) / kSmoothRows);
        k_smooth_am_rows<<<aparts, kRowThreads, 0, s>>>(m, dam);
        count_launch();
        k_smooth_G<<<(m.V + kRowThreads - 1) / kRowThreads, kRowThreads, 0, s>>>(m, aparts);
        count_launch();
    }
    k_smooth_lm_rows_bwd<<<row_grid(lrows, kRowThreads / 32), kRowThreads, 0, s>>>(m, dlm);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_prune_ranges(cudaStream_t s, const float2 *pg, const float *raw_blank, const int *xn, const int *yn,
                                int N, int T, int U, int S, int rnnt_type, int *ranges) {
    if (rnnt_type == 2) k_prune_ranges<2><<<N, kRangeThreads, 0, s>>>(pg, xn, yn, T, U, S, ranges, raw_blank);
    else if (rnnt_type == 1) k_prune_ranges<1><<<N, kRangeThreads, 0, s>>>(pg, xn, yn, T, U, S, ranges, nullptr);
    else k_prune_ranges<0><<<N, kRangeThreads, 0, s>>>(pg, xn, yn, T, U, S, ranges, nullptr);
    count_launch();
    return cudaGetLastError();
}

}  // namespace rnnt
