// joint.cu -- compact packing of the joint network's input (SURVEY.md 8(f)3): the caller side of compact=True.
//
// The reference's benchmark builds the ragged joint input with a python loop over the batch
// (the reference's pytorch_binding/benchmark2.py:37-50):
//     x = cat([ (f[i, :lf[i]].unsqueeze(1) + g[i, :lg[i]+1].unsqueeze(0)).view(-1, H)  for i in range(N) ])
// i.e. 2N host syncs (lf[i], lg[i] index tensors), N small kernels + a cat, and autograd replays the same pieces
// backwards.  Here: one kernel forward (rows at mem_pref[n] + t*(lg[n]+1) + u, the layout rnnt_loss(compact=True)
// expects), two deterministic reduction kernels backward, no host sync when the caller passes STU.
//   x[row(n,t,u), :] = f[n,t,:] + g[n,u,:]                       t < lf[n], u <= lg[n]
//   df[n,t,:] = sum_u dx[row(n,t,u), :]   (0 for t >= lf[n])     dg[n,u,:] = sum_t dx[row(n,t,u), :]   (0 for u > lg[n])
// All three are pure streaming: bytes = 4*H per packed row written (forward) or read twice (backward).
#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

constexpr int kJointThreads = 256;

// grid (chunks, N): a CTA walks the cells of lattice n.  L = min(H/VEC, 256) threads cover one packed row's h-vectors,
// R = 256 / L rows per pass; the (t, u) of a thread's row advances by a running cursor (one division per thread).
template <int VEC>
__global__ void __launch_bounds__(kJointThreads)
k_joint_pack(const float *__restrict__ f, const float *__restrict__ g, const int *__restrict__ lf,
             const int *__restrict__ lg, const int64_t *__restrict__ mem_pref, float *__restrict__ x, int T, int U1,
             int H) {
    const int n = blockIdx.y;
    const int Tn = lf[n], Un = lg[n] + 1;
    if (Tn < 1 || Tn > T || Un < 1 || Un > U1) return;
    const int hv = H / VEC;                                 // vectors per row
    const int L = min(hv, kJointThreads), R = kJointThreads / L;
    const int r = threadIdx.x / L, l = threadIdx.x - r * L;
    if (r >= R) return;                                     // (256 % L) surplus threads
    const int cells = Tn * Un;
    const int stride = gridDim.x * R;                       // cells per pass of the grid
    int cell = blockIdx.x * R + r;
    int t = cell / Un, u = cell - t * Un;
    const int dt = stride / Un, du = stride - dt * Un;
    const float *fn = f + (int64_t)n * T * H, *gn = g + (int64_t)n * U1 * H;
    float *xn = x + mem_pref[n] * H;
    for (; cell < cells; cell += stride) {
        const float *fr = fn + (int64_t)t * H, *gr = gn + (int64_t)u * H;
        float *dst = xn + (int64_t)cell * H;
        for (int q = l; q < hv; q += L) {
            if (VEC == 4) {
                const float4 a = __ldg(reinterpret_cast<const float4 *>(fr) + q);
                const float4 b = __ldg(reinterpret_cast<const float4 *>(gr) + q);
                st_cs_v4(dst + 4 * q, make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w));
            } else {
                st_cs(dst + q, __ldg(fr + q) + __ldg(gr + q));
            }
        }
        t += dt; u += du;
        if (u >= Un) { u -= Un; ++t; }
    }
}

// df: grid (T, N); a CTA sums the Un packed rows of (n,t): contiguous Un*H floats.  Threads own h-vectors.
template <int VEC>
__global__ void __launch_bounds__(kJointThreads)
k_joint_grad_f(const float *__restrict__ dx, const int *__restrict__ lf, const int *__restrict__ lg,
               const int64_t *__restrict__ mem_pref, float *__restrict__ df, int T, int U1, int H) {
    const int n = blockIdx.y, t = blockIdx.x;
    const int Tn = lf[n], Un = lg[n] + 1;
    const bool live = (Tn >= 1 && Tn <= T && Un >= 1 && Un <= U1 && t < Tn);
    float *out = df + ((int64_t)n * T + t) * H;
    const float *src = live ? dx + (mem_pref[n] + (int64_t)t * Un) * H : nullptr;
    for (int h = threadIdx.x * VEC; h < H; h += kJointThreads * VEC) {
        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = 0.0f;
        if (live) {
            for (int u = 0; u < Un; ++u) {                  // fixed order: deterministic
                if (VEC == 4) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(src + (int64_t)u * H + h));
                    acc[0] += v.x; acc[1 % VEC] += v.y; acc[2 % VEC] += v.z; acc[3 % VEC] += v.w;
                } else {
                    acc[0] += __ldg(src + (int64_t)u * H + h);
                }
            }
        }
        if (VEC == 4) *reinterpret_cast<float4 *>(out + h) = make_float4(acc[0], acc[1 % VEC], acc[2 % VEC], acc[3 % VEC]);
        else out[h] = acc[0];
    }
}

// dg: grid (U1, N); a CTA sums over t the rows (n,t,u): stride Un*H between them.
template <int VEC>
__global__ void __launch_bounds__(kJointThreads)
k_joint_grad_g(const float *__restrict__ dx, const int *__restrict__ lf, const int *__restrict__ lg,
               const int64_t *__restrict__ mem_pref, float *__restrict__ dg, int T, int U1, int H) {
    const int n = blockIdx.y, u = blockIdx.x;
    const int Tn = lf[n], Un = lg[n] + 1;
    const bool live = (Tn >= 1 && Tn <= T && Un >= 1 && Un <= U1 && u < Un);
    float *out = dg + ((int64_t)n * U1 + u) * H;
    const float *src = live ? dx + (mem_pref[n] + u) * H : nullptr;
    const int64_t step = (int64_t)Un * H;
    for (int h = threadIdx.x * VEC; h < H; h += kJointThreads * VEC) {
        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = 0.0f;
        if (live) {
            for (int t = 0; t < Tn; ++t) {
                if (VEC == 4) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(src + t * step + h));
                    acc[0] += v.x; acc[1 % VEC] += v.y; acc[2 % VEC] += v.z; acc[3 % VEC] += v.w;
                } else {
                    acc[0] += __ldg(src + t * step + h);
                }
            }
        }
        if (VEC == 4) *reinterpret_cast<float4 *>(out + h) = make_float4(acc[0], acc[1 % VEC], acc[2 % VEC], acc[3 % VEC]);
        else out[h] = acc[0];
    }
}

static bool vec4_ok(const void *a, const void *b, const void *c, int H) {
    return (H % 4 == 0) && (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15u) == 0);
}

cudaError_t launch_joint_pack(cudaStream_t s, const float *f, const float *g, const int *lf, const int *lg,
                              const int64_t *mem_pref, float *x, int N, int T, int U1, int H, int64_t stu_hint) {
    if (N <= 0) return cudaSuccess;
    const int sms = sm_count(current_device());
    const bool v4 = vec4_ok(f, g, x, H);
    const int hv = H / (v4 ? 4 : 1), rows_per_cta = kJointThreads / min(hv, kJointThreads);
    const int64_t per = stu_hint > 0 ? stu_hint / N + 1 : (int64_t)T * U1;     // cells per lattice (estimate)
    int gx = (int)min((per + rows_per_cta * 4 - 1) / (rows_per_cta * 4), (int64_t)max(1, sms * 8 / N));
    gx = max(gx, 1);
    dim3 grid(gx, N);
    if (v4) k_joint_pack<4><<<grid, kJointThreads, 0, s>>>(f, g, lf, lg, mem_pref, x, T, U1, H);
    else k_joint_pack<1><<<grid, kJointThreads, 0, s>>>(f, g, lf, lg, mem_pref, x, T, U1, H);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_joint_grads(cudaStream_t s, const float *dx, const int *lf, const int *lg, const int64_t *mem_pref,
                               float *df, float *dg, int N, int T, int U1, int H) {
    if (N <= 0) return cudaSuccess;
    const bool v4 = vec4_ok(dx, df, dg, H);
    if (df) {
        dim3 grid(T, N);
        if (v4) k_joint_grad_f<4><<<grid, kJointThreads, 0, s>>>(dx, lf, lg, mem_pref, df, T, U1, H);
        else k_joint_grad_f<1><<<grid, kJointThreads, 0, s>>>(dx, lf, lg, mem_pref, df, T, U1, H);
        count_launch();
    }
    if (dg) {
        dim3 grid(U1, N);
        if (v4) k_joint_grad_g<4><<<grid, kJointThreads, 0, s>>>(dx, lf, lg, mem_pref, dg, T, U1, H);
        else k_joint_grad_g<1><<<grid, kJointThreads, 0, s>>>(dx, lf, lg, mem_pref, dg, T, U1, H);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace rnnt
