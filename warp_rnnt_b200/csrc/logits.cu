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
#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kLogitThreads = 256;

// SUB lanes cooperate on one cell (SUB in {1, 8, 32}); online max / sum so the row is read once.  VEC4: rows are whole
// float4s at 16-byte aligned addresses -> the SUB lanes stride over float4s (V = 28: 7 of 8 lanes load one vector each,
// a warp reads 4 consecutive rows = 448 contiguous bytes).
template <int SUB, bool VEC4>
__global__ void __launch_bounds__(kLogitThreads)
k_lse_pairs(const float *__restrict__ x, const int *__restrict__ labels, int64_t cells, int V, int blank, int U,
            FastDiv divU, FastDiv divTU, float2 *__restrict__ pairs, float *__restrict__ lse_out) {
    const int sub = threadIdx.x % SUB;
    const int64_t per_block = kLogitThreads / SUB;
    for (int64_t base = (int64_t)blockIdx.x * per_block; base < cells; base += (int64_t)gridDim.x * per_block) {   // block-uniform trip count
        const int64_t cell = min(base + threadIdx.x / SUB, cells - 1);          // surplus groups redo the last cell (shuffles need every lane)
        const float *row = x + cell * V;
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
            // the whole row is one float4 per lane: max first (shuffles only), then ONE exp per element -- the online
            // merge below would spend two more exp per lane and shuffle round
            const bool has = sub < (V >> 2);
            const float4 a = has ? __ldg(reinterpret_cast<const float4 *>(row) + sub) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            m = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            s = has ? (expf(a.x - m) + expf(a.y - m)) + (expf(a.z - m) + expf(a.w - m)) : 0.0f;
#pragma unroll
            for (int o = SUB / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        } else if (VEC4) {
            const float4 *row4 = reinterpret_cast<const float4 *>(row);
            for (int q = sub; q < (V >> 2); q += SUB) {
                const float4 a = __ldg(row4 + q);
                const float mx = fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w));
                if (mx > m) { s = s * expf(m - mx); m = mx; }
                const float mo = off();
                s += (expf(a.x - mo) + expf(a.y - mo)) + (expf(a.z - mo) + expf(a.w - mo));
            }
        } else if (SUB == 1) {
            // short unaligned rows: one thread per cell; neighbouring threads' rows share cache lines, so the pass over
            // v is served from L1 after the first touch
            for (int v = 0; v < V; ++v) m = fmaxf(m, __ldg(row + v));
            for (int v = 0; v < V; ++v) s += expf(__ldg(row + v) - m);
        } else {
            for (int v = sub; v < V; v += SUB) add(__ldg(row + v));
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
            uint32_t n, rem, t, u;
            divTU.divmod((uint32_t)cell, n, rem);
            divU.divmod(rem, t, u);
            const int lab = ((int)u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : blank;
            pairs[cell] = make_float2(__ldg(row + blank) - l, __ldg(row + lab) - l);
            lse_out[cell] = l;
        }
    }
}

// flat stream of the (cells, V) output in vectors of VEC floats (VEC = 4 when V % 4 == 0, 2 when V % 2 == 0, else 1):
// a vector never straddles a row, so one (gb, gl, lse, label) fetch serves it.
template <int VEC>
__global__ void __launch_bounds__(kLogitThreads)
k_expand_logits(const float *__restrict__ x, const float *__restrict__ lse, const float2 *__restrict__ pg,
                const int *__restrict__ labels, const float *__restrict__ grad_out, float *__restrict__ out,
                int64_t cells, int V, int blank, int U, FastDiv divU, FastDiv divTU, int64_t stride_rows,
                int stride_v) {
    const int64_t total = cells * (int64_t)V;
    int64_t f = ((int64_t)blockIdx.x * kLogitThreads + threadIdx.x) * VEC;
    if (f >= total) return;
    // (row, v0) of the thread's vector: one 64-bit division here, then a running cursor (the grid stride is
    // stride_rows whole rows + stride_v floats)
    int64_t row = f / V;
    int v0 = (int)(f - row * V);
    const int64_t stride = stride_rows * V + stride_v;
    for (; f < total; f += stride, row += stride_rows, v0 += stride_v) {
        if (v0 >= V) { v0 -= V; ++row; }
        const float2 q = pg[row];
        float e[VEC];
        if (q.x == 0.0f && q.y == 0.0f) {
            // padding (or a cell without gradient): exact zeros -- (0 - softmax * 0), as log_softmax's backward gives,
            // which is NaN when the row's normaliser is NaN (a NaN or +inf logit, or every logit -inf)
            const float z = (lse[row] == lse[row]) ? 0.0f : NAN;
#pragma unroll
            for (int k = 0; k < VEC; ++k) e[k] = z;
        } else {
            uint32_t n, rem, t, u;
            divTU.divmod((uint32_t)row, n, rem);
            divU.divmod(rem, t, u);
            const int lab = ((int)u < U - 1) ? labels[(int64_t)n * (U - 1) + u] : -1;
            const float sc = grad_out ? grad_out[n] : 1.0f;
            const float l = lse[row], tot = q.x + q.y;
            float xv[VEC];
            if (VEC == 4) {
                const float4 t4 = __ldg(reinterpret_cast<const float4 *>(x + f));
                xv[0] = t4.x; xv[1] = t4.y; xv[2 % VEC] = t4.z; xv[3 % VEC] = t4.w;
            } else if (VEC == 2) {
                const float2 t2 = __ldg(reinterpret_cast<const float2 *>(x + f));
                xv[0] = t2.x; xv[1 % VEC] = t2.y;
            } else {
                xv[0] = __ldg(x + f);
            }
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                float gsel = (v0 + k == blank) ? q.x : 0.0f;
                if (v0 + k == lab) gsel += q.y;
                e[k] = (gsel - expf(xv[k] - l) * tot) * sc;
            }
        }
        if (VEC == 4) st_cs_v4(out + f, make_float4(e[0], e[1 % VEC], e[2 % VEC], e[3 % VEC]));
        else if (VEC == 2) st_cs_v2(out + f, make_float2(e[0], e[1 % VEC]));
        else st_cs(out + f, e[0]);
    }
}

cudaError_t launch_lse_pairs(cudaStream_t s, const float *x, const int *labels, int N, int T, int U, int V, int blank,
                             float2 *pairs, float *lse) {
    const int64_t cells = (int64_t)N * T * U;
    if (cells <= 0) return cudaSuccess;
    const FastDiv divU((uint32_t)U), divTU((uint32_t)(T * U));
    const int sms = sm_count(current_device());
    const bool vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15u) == 0);
    const int sub = vec4 ? (V <= 32 ? 8 : 32) : (V <= 12 ? 1 : (V <= 512 ? 8 : 32));
    const int64_t per_block = kLogitThreads / sub;
    const int grid = (int)min((cells + per_block - 1) / per_block, (int64_t)sms * 16);
#define RNNT_LSE_LAUNCH(SUB, VEC) k_lse_pairs<SUB, VEC><<<grid, kLogitThreads, 0, s>>>(x, labels, cells, V, blank, U, divU, divTU, pairs, lse)
    if (vec4) { if (sub == 8) RNNT_LSE_LAUNCH(8, true); else RNNT_LSE_LAUNCH(32, true); }
    else if (sub == 1) RNNT_LSE_LAUNCH(1, false);
    else if (sub == 8) RNNT_LSE_LAUNCH(8, false);
    else RNNT_LSE_LAUNCH(32, false);
#undef RNNT_LSE_LAUNCH
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_expand_logits(cudaStream_t s, const float *x, const float *lse, const float2 *pg, const int *labels,
                                 const float *grad_out, float *out, int N, int T, int U, int V, int blank) {
    const int64_t cells = (int64_t)N * T * U;
    if (cells <= 0) return cudaSuccess;
    const FastDiv divU((uint32_t)U), divTU((uint32_t)(T * U));
    const int sms = sm_count(current_device());
    const bool al16 = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0;
    const bool al8 = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 7u) == 0;
    const int vec = (V % 4 == 0 && al16) ? 4 : ((V % 2 == 0 && al8) ? 2 : 1);
    const int64_t total = cells * (int64_t)V / vec;
    const int grid = (int)min((total + kLogitThreads - 1) / kLogitThreads, (int64_t)sms * 32);
    const int64_t stride = (int64_t)grid * kLogitThreads * vec;
    const int64_t srows = stride / V;
    const int sv = (int)(stride - srows * V);
    if (vec == 4) k_expand_logits<4><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv);
    else if (vec == 2) k_expand_logits<2><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv);
    else k_expand_logits<1><<<grid, kLogitThreads, 0, s>>>(x, lse, pg, labels, grad_out, out, cells, V, blank, U, divU, divTU, srows, sv);
    count_launch();
    return cudaGetLastError();
}

}  // namespace rnnt
