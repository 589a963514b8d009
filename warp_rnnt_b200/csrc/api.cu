// api.cu -- the extern "C" surface of librnnt_b200.so (declared in include/rnnt_b200.h).
//
// (A) rnnt_b200_*: native interface bound by csrc/binding.cpp.
// (B) run_warp_rnnt & co: the reference's C ABI (the reference's core.h:29-60) implemented on top
//     of (A)'s kernels so the reference's own bindings link against this library unchanged.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

static std::atomic<int> g_poison_n{-1};
static std::atomic<float> g_poison_delta{0.0f};
GuardPoison guard_poison() { return {g_poison_n.load(std::memory_order_relaxed), g_poison_delta.load(std::memory_order_relaxed)}; }

static int env_lse_mode() {
    const char *e = getenv("RNNT_B200_LSE");
    if (!e) return RNNT_LSE_AUTO;
    if (!strcmp(e, "exact")) return RNNT_LSE_EXACT;
    if (!strcmp(e, "fast")) return RNNT_LSE_FAST;
    return RNNT_LSE_AUTO;
}
static std::atomic<int> g_lse_mode{-1};

static int default_lse_mode() {
    int m = g_lse_mode.load(std::memory_order_relaxed);
    if (m < 0) {
        m = env_lse_mode();
        g_lse_mode.store(m, std::memory_order_relaxed);
    }
    return m;
}

// AUTO policy (DESIGN.md "numerics"): AUTO = exact, i.e. results are bit-identical to the reference
// kernels unless the caller opts out.  Parity is the first gate: at BASELINE cfg 2 the fast flavour
// differs from the reference by fp32 noise that can exceed the stated 1e-4 on single gradient elements (the
// full-size test bounds it at 2.5e-4).  The exact chain is ~2x longer per anti-diagonal, but on an H100
// (700 W) the dense cfg-2 call takes 110 us in both flavours: the dense gradient write dominates.
// RNNT_LSE_FAST / RNNT_B200_LSE=fast selects the short chain.
static int resolve_kind(int lse_mode, bool compact) {
    if (lse_mode == RNNT_LSE_AUTO) lse_mode = default_lse_mode();
    if (lse_mode == RNNT_LSE_FAST) return kFast;
    return compact ? kExactCompact : kExactDense;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// RNNT_B200_PATH = auto | fused | general  (tests exercise both paths on the same inputs)
static int forced_path() {
    static const int path = [] {
        const char *e = getenv("RNNT_B200_PATH");
        return (e && !strcmp(e, "general")) ? 2 : (e && !strcmp(e, "fused")) ? 1 : 0;
    }();
    return path;
}
static bool want_fused(int N, int T, int U, FusedPlan *plan) {
    if (forced_path() >= 2) return false;
    return fused_plan(N, T, U, plan);
}

struct Workspace {
    float2 *pairs;
    float *alphas, *betas, *ll;
    int *bad;
    int64_t *mem_pref, *lab_pref;
    int *totals;
    size_t bytes;
};

static Workspace carve(void *base, int64_t cells, int N) {
    Workspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void *p = base ? (void *)((char *)base + off) : nullptr;
        off += align_up(bytes, 256);
        return p;
    };
    const size_t c = (size_t)(cells > 0 ? cells : 0), n = (size_t)(N > 0 ? N : 0);
    w.pairs = (float2 *)take(c * sizeof(float2));
    w.alphas = (float *)take(c * sizeof(float));
    w.betas = (float *)take(c * sizeof(float));
    w.ll = (float *)take(2 * n * sizeof(float));
    w.bad = (int *)take(n * sizeof(int));
    w.mem_pref = (int64_t *)take(n * sizeof(int64_t));
    w.lab_pref = (int64_t *)take(n * sizeof(int64_t));
    w.totals = (int *)take(4 * sizeof(int));
    w.bytes = off;
    return w;
}

static bool dense_args_ok(int N, int T, int U, int V) {
    if (N < 0 || T < 1 || U < 1 || V < 1) return false;
    if ((int64_t)T * U >= (int64_t)1 << 31) return false;
    if ((int64_t)N * T * U >= (int64_t)1 << 31) return false;   // cell ids are 32-bit in the emit kernel
    if (V >= (1 << 22)) return false;
    return true;
}

// Internal streams for the pipelined general path: one for gathers, one for emits, four
// high-priority ones for wavefronts (their CTAs are few and long-lived; priority lets them take the
// SMs that free up at every gather / emit kernel boundary).  Created once per process and device.
struct Pipeline {
    static constexpr int kWave = 4, kGroups = 8;
    cudaStream_t gather_s, expand_s, wave_s[kWave];
    cudaEvent_t fork, gathered[kGroups], swept[kGroups], join[2 + kWave];
    int device;
};
static bool pipeline_enabled() {
    // on by default (RNNT_B200_PIPELINE=0 disables).  It only pays off with the early-retiring emit grid
    // (launch_expand retire_early): persistent emit CTAs hold every SM until their kernel ends and the
    // high-priority wavefront CTAs never get in.
    static const bool on = !env_is("RNNT_B200_PIPELINE", '0');
    return on;
}
// One pipeline per device (streams and events belong to a device); created on first use under g_pipe_mu,
// which also serialises the calls that use a pipeline's shared events.
static std::mutex g_pipe_mu;
static Pipeline *get_pipeline_locked() {
    static Pipeline *pipes[kMaxDevices] = {};
    const int dev = current_device();
    if (dev >= kMaxDevices) return nullptr;
    if (pipes[dev]) return pipes[dev];
    Pipeline *p = new Pipeline();
    p->device = dev;
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);  // hi = numerically lowest = highest priority
    bool ok = cudaStreamCreateWithPriority(&p->gather_s, cudaStreamNonBlocking, lo) == cudaSuccess &&
              cudaStreamCreateWithPriority(&p->expand_s, cudaStreamNonBlocking, lo) == cudaSuccess;
    for (int i = 0; i < Pipeline::kWave && ok; ++i)
        ok = cudaStreamCreateWithPriority(&p->wave_s[i], cudaStreamNonBlocking, hi) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&p->fork, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < Pipeline::kGroups && ok; ++i)
        ok = cudaEventCreateWithFlags(&p->gathered[i], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&p->swept[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < 2 + Pipeline::kWave && ok; ++i)
        ok = cudaEventCreateWithFlags(&p->join[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { cudaGetLastError(); delete p; return nullptr; }
    pipes[dev] = p;
    return p;
}

// Self-check of the restated log1pf (common.cuh:log1pf_unit) against libdevice: every float in [+0, 1], a NaN, and the
// complete exact LSE (both flavours) on pseudo-random operand pairs.  counts[0] += mismatches.
__global__ void k_lse_selfcheck(unsigned long long *counts) {
    unsigned long long bad = 0;
    const uint32_t top = 0x3f800000u;                       // 1.0f
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b <= top; b += (uint64_t)gridDim.x * blockDim.x) {
        const float x = __uint_as_float((uint32_t)b);
        const uint32_t r0 = __float_as_uint(log1pf(x)), r1 = __float_as_uint(log1pf_unit(x));
        bad += (r0 != r1);
    }
    // NaN in, NaN out (the guard lives in lse_tail); NaN / inf - inf operands of the whole LSE stay NaN like the reference's
    { const float n = lse_tail(-1.0f, __uint_as_float(0x7fc00000u + threadIdx.x)); bad += !(n != n); }
    {
        const float qn = __uint_as_float(0x7fc00000u), inf = __uint_as_float(0x7f800000u);
        const float A4[8] = {qn, 1.0f, -inf, inf, -3.0f, 0.0f, -inf, -2.5f}, B4[8] = {1.0f, qn, -inf, inf, -3.0f, -0.0f, -7.0f, -inf};
        for (int k = 0; k < 8; ++k) {
            const float a = A4[k], b2 = B4[k];
            float mx, df;
            if (a > b2) { mx = a; df = b2 - a; } else { mx = b2; df = a - b2; }
            const float ref = mx + log1pf(expf(df)), got = lse<kExactDense>(a, b2);
            bad += ((ref != ref) != (got != got)) || (ref == ref && __float_as_uint(ref) != __float_as_uint(got));
            const float tmp = a - b2;
            const float refc = (a == b2) ? (float)(a + M_LN2) : (tmp > 0) ? a + log1pf(expf(-tmp)) : (tmp <= 0) ? b2 + log1pf(expf(tmp)) : tmp;
            const float gotc = lse<kExactCompact>(a, b2);
            bad += ((refc != refc) != (gotc != gotc)) || (refc == refc && __float_as_uint(refc) != __float_as_uint(gotc));
        }
    }
    // -0 as the larger operand: (-0) + log1p(e) and (+0) + log1p(e) are the same float for every e in [0, 1]
    { const float r0 = lse<kExactDense>(-0.0f, -3.0f), r1 = -0.0f + log1pf(expf(-3.0f)); bad += (__float_as_uint(r0) != __float_as_uint(r1));
      const float r2 = lse<kExactDense>(-0.0f, -__uint_as_float(0x7f800000u)), r3 = -0.0f + log1pf(0.0f); bad += (__float_as_uint(r2) != __float_as_uint(r3)); }
    // the whole LSE on operand pairs spread over the magnitudes the lattices see (a hash of the thread index)
    uint32_t h = 0x9e3779b9u * ((uint32_t)blockIdx.x * blockDim.x + threadIdx.x + 1u);
    for (int k = 0; k < 64; ++k) {
        h = h * 1664525u + 1013904223u;
        const float a = -(float)(h >> 8) * (1.0f / 65536.0f) * 40.0f;       // [-10240, 0]
        h = h * 1664525u + 1013904223u;
        const float d = ((float)(h >> 8) * (1.0f / 16777216.0f) - 0.5f) * ((k & 1) ? 40.0f : 2.0f);
        const float b2 = a + d;
        float mx, df;
        if (a > b2) { mx = a; df = b2 - a; } else { mx = b2; df = a - b2; }
        const float ref = mx + log1pf(expf(df));
        bad += (__float_as_uint(ref) != __float_as_uint(lse<kExactDense>(a, b2)));
        const float tmp = a - b2;
        float refc = (a == b2) ? (float)(a + M_LN2) : ((tmp > 0) ? a + log1pf(expf(-tmp)) : b2 + log1pf(expf(tmp)));
        bad += (__float_as_uint(refc) != __float_as_uint(lse<kExactCompact>(a, b2)));
    }
    if (bad) atomicAdd(counts, bad);
}

#define RNNT_TRY(expr, code)                                            \
    do {                                                                \
        cudaError_t e__ = (expr);                                       \
        if (e__ != cudaSuccess) {                                       \
            fprintf(stderr, "rnnt_b200: %s failed: %s\n", #expr, cudaGetErrorString(e__)); \
            return (code);                                              \
        }                                                               \
    } while (0)

}  // namespace rnnt

using namespace rnnt;

// dense layout, log_probs / grads of 4-byte (f32) or 2-byte (bf16) elements
static int loss_dense_any(void *stream, void *workspace, size_t workspace_bytes, const void *log_probs,
                          const int *labels, const int *xn, const int *yn, float *costs, void *grads,
                          const float *grad_scale, float *loss_sum, unsigned int *sync_counter, int N, int T,
                          int U, int V, int blank, float fastemit_lambda, int lse_mode, int io_bf16) {
    const size_t esz = io_bf16 ? 2 : 4;
    auto lp_at = [&](int64_t cell0) { return (const void *)((const char *)log_probs + (size_t)cell0 * V * esz); };
    auto g_at = [&](int64_t cell0) { return (void *)((char *)grads + (size_t)cell0 * V * esz); };
    if (io_bf16 && !grads) return RNNT_STATUS_INVALID_ARGUMENT;
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    FusedPlan plan;
    if (want_fused(N, T, U, &plan)) {
        RNNT_TRY(launch_fused(s, resolve_kind(lse_mode, false), plan, log_probs, labels, xn, yn, costs, grads, nullptr,
                              grad_scale, N, T, U, V, blank, fastemit_lambda, 0, 1, nullptr, nullptr, nullptr, loss_sum,
                              sync_counter, io_bf16),
                 RNNT_STATUS_WARP_FAILED);
        if (loss_sum && !sync_counter)                  // no counter: reduce in a second, tiny launch
            RNNT_TRY(launch_loss_sum(s, costs, grad_scale, N, loss_sum), RNNT_STATUS_COSTS_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    const Workspace w = carve(workspace, cells, N);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    const int kind = resolve_kind(lse_mode, false);
    // Large batches of large lattices: software-pipeline lattice groups over internal streams so that the
    // latency-bound wavefront of group g overlaps the bandwidth-bound gather of g+1 and emit of g-1.
    // ... which only pays when the wavefront (a per-lattice latency chain of T+U-1 steps that does not shrink with the
    // group) is short against the bandwidth-bound emit: cfg 5's micro-batch takes the pipeline, cfg 4 does not.
    // The two estimates (0.45 us per anti-diagonal, an emit at 5.5 TB/s) were measured on a B200 and have not been
    // re-derived for the H100 (3.35 TB/s HBM3): there the emit is slower, so the true break-even favours the pipeline more often than this estimate.
    const double wave_us = 0.45 * (T + U), emit_us = (double)cells * V * (io_bf16 ? 2 : 4) / 5.5e6;
    const int groups = (grads && N >= 8 && (int64_t)cells * V * 4 >= ((int64_t)512 << 20) && pipeline_enabled() &&
                        wave_us < 0.4 * emit_us)
                           ? (N >= 32 ? 8 : 4) : 1;
    if (groups > 1) {
        std::lock_guard<std::mutex> lock(g_pipe_mu);    // the pipeline's events are shared by all calls on this device
        Pipeline *pl = get_pipeline_locked();
        if (pl) {
            int status = RNNT_STATUS_SUCCESS;
            cudaEventRecord(pl->fork, s);
            cudaStreamWaitEvent(pl->gather_s, pl->fork, 0);
            cudaStreamWaitEvent(pl->expand_s, pl->fork, 0);
            for (int i = 0; i < Pipeline::kWave; ++i) cudaStreamWaitEvent(pl->wave_s[i], pl->fork, 0);
            for (int g = 0; g < groups && !status; ++g) {
                const int n0 = (int)((int64_t)N * g / groups), n1 = (int)((int64_t)N * (g + 1) / groups);
                const int ng = n1 - n0;
                const int64_t c0 = (int64_t)n0 * T * U, cg = (int64_t)ng * T * U;
                Problem p = {xn + n0, yn + n0, nullptr, nullptr, ng, T, U, 0};
                const int *lab_g = labels + (int64_t)n0 * (U - 1);
                cudaStream_t ws = pl->wave_s[g % Pipeline::kWave];
                if (launch_gather(pl->gather_s, p, lp_at(c0), lab_g, V, blank, w.pairs + c0, nullptr, cg, io_bf16) != cudaSuccess)
                    status = RNNT_STATUS_GATHER_FAILED;
                cudaEventRecord(pl->gathered[g], pl->gather_s);
                cudaStreamWaitEvent(ws, pl->gathered[g], 0);
                if (!status && launch_wavefront(ws, kind, p, w.pairs + c0, w.alphas + c0, w.betas + c0, w.ll + 2 * n0,
                                                w.bad + n0, costs + n0, 0, 1, T, U) != cudaSuccess)
                    status = RNNT_STATUS_WARP_FAILED;
                cudaEventRecord(pl->swept[g], ws);
                cudaStreamWaitEvent(pl->expand_s, pl->swept[g], 0);
                ExpandSrc src = {};
                src.pairs = w.pairs + c0; src.alphas = w.alphas + c0; src.betas = w.betas + c0; src.bad = w.bad + n0;
                src.scale = grad_scale ? grad_scale + n0 : nullptr; src.labels = lab_g; src.fastemit_lambda = fastemit_lambda;
                if (!status && launch_expand(pl->expand_s, p, src, g_at(c0), cg, V, blank, true, io_bf16) != cudaSuccess)
                    status = RNNT_STATUS_GRADS_BLANK_FAILED;
            }
            cudaEventRecord(pl->join[0], pl->gather_s);
            cudaEventRecord(pl->join[1], pl->expand_s);
            cudaStreamWaitEvent(s, pl->join[0], 0);
            cudaStreamWaitEvent(s, pl->join[1], 0);
            for (int i = 0; i < Pipeline::kWave; ++i) {
                cudaEventRecord(pl->join[2 + i], pl->wave_s[i]);
                cudaStreamWaitEvent(s, pl->join[2 + i], 0);
            }
            if (!status && loss_sum && launch_loss_sum(s, costs, grad_scale, N, loss_sum) != cudaSuccess)
                status = RNNT_STATUS_COSTS_FAILED;
            return status;
        }
    }
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    RNNT_TRY(launch_gather(s, p, log_probs, labels, V, blank, w.pairs, nullptr, cells, io_bf16), RNNT_STATUS_GATHER_FAILED);
    RNNT_TRY(launch_wavefront(s, kind, p, w.pairs, w.alphas, w.betas, w.ll, w.bad, costs, grads == nullptr, 1, T, U),
             RNNT_STATUS_WARP_FAILED);
    if (grads) {
        ExpandSrc src = {};
        src.pairs = w.pairs; src.alphas = w.alphas; src.betas = w.betas; src.bad = w.bad;
        src.scale = grad_scale; src.labels = labels; src.fastemit_lambda = fastemit_lambda;
        RNNT_TRY(launch_expand(s, p, src, grads, cells, V, blank, false, io_bf16), RNNT_STATUS_GRADS_BLANK_FAILED);
    }
    if (loss_sum) RNNT_TRY(launch_loss_sum(s, costs, grad_scale, N, loss_sum), RNNT_STATUS_COSTS_FAILED);
    return RNNT_STATUS_SUCCESS;
}


extern "C" {

const char *rnnt_b200_version(void) { return "0.1.0 (sm_90a)"; }

const char *rnnt_b200_status_string(int s) {
    switch (s) {
        case RNNT_STATUS_SUCCESS: return "success";
        case RNNT_STATUS_WARP_FAILED: return "alpha/beta wavefront kernel failed";
        case RNNT_STATUS_GRADS_BLANK_FAILED: return "gradient kernel failed";
        case RNNT_STATUS_GRADS_LABEL_FAILED: return "gradient kernel (label) failed";
        case RNNT_STATUS_COSTS_FAILED: return "cost kernel failed";
        case RNNT_STATUS_INVALID_ARGUMENT: return "invalid argument";
        case RNNT_STATUS_WORKSPACE_TOO_SMALL: return "workspace too small";
        case RNNT_STATUS_GATHER_FAILED: return "gather kernel failed";
        default: return "unknown status";
    }
}

void rnnt_b200_set_lse_mode(int mode) {
    if (mode < RNNT_LSE_AUTO || mode > RNNT_LSE_FAST) mode = RNNT_LSE_AUTO;
    g_lse_mode.store(mode, std::memory_order_relaxed);
}
int rnnt_b200_get_lse_mode(void) { return default_lse_mode(); }

uint64_t rnnt_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
void rnnt_b200_debug_guard_poison(int n, float delta) {
    g_poison_delta.store(delta, std::memory_order_relaxed);
    g_poison_n.store(n, std::memory_order_relaxed);
}
int rnnt_b200_debug_lse_selfcheck(void *stream, unsigned long long *mismatches) {
    if (!mismatches) return RNNT_STATUS_INVALID_ARGUMENT;
    rnnt::k_lse_selfcheck<<<sm_count(current_device()) * 8, 256, 0, (cudaStream_t)stream>>>(mismatches);
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_WARP_FAILED;
}
void rnnt_b200_debug_fused_trace(void *buf) { rnnt::set_fused_trace(static_cast<long long *>(buf)); }

size_t rnnt_b200_workspace_bytes(int64_t cells, int N) { return carve(nullptr, cells, N).bytes; }

int rnnt_b200_loss_dense(void *stream, void *workspace, size_t workspace_bytes, const float *log_probs,
                         const int *labels, const int *xn, const int *yn, float *costs, float *grads,
                         const float *grad_scale, int N, int T, int U, int V, int blank, float fastemit_lambda,
                         int lse_mode) {
    return rnnt_b200_loss_dense_reduced(stream, workspace, workspace_bytes, log_probs, labels, xn, yn, costs, grads,
                                        grad_scale, nullptr, nullptr, N, T, U, V, blank, fastemit_lambda, lse_mode);
}

int rnnt_b200_loss_dense_reduced(void *stream, void *workspace, size_t workspace_bytes, const float *log_probs,
                                 const int *labels, const int *xn, const int *yn, float *costs, float *grads,
                                 const float *grad_scale, float *loss_sum, unsigned int *sync_counter, int N, int T,
                                 int U, int V, int blank, float fastemit_lambda, int lse_mode) {
    return loss_dense_any(stream, workspace, workspace_bytes, log_probs, labels, xn, yn, costs, grads, grad_scale,
                          loss_sum, sync_counter, N, T, U, V, blank, fastemit_lambda, lse_mode, 0);
}

int rnnt_b200_loss_dense_bf16(void *stream, void *workspace, size_t workspace_bytes, const void *log_probs_bf16,
                              const int *labels, const int *xn, const int *yn, float *costs, void *grads_bf16,
                              const float *grad_scale, float *loss_sum, unsigned int *sync_counter, int N, int T,
                              int U, int V, int blank, float fastemit_lambda, int lse_mode) {
    if ((reinterpret_cast<uintptr_t>(log_probs_bf16) | reinterpret_cast<uintptr_t>(grads_bf16)) & 1u)
        return RNNT_STATUS_INVALID_ARGUMENT;
    return loss_dense_any(stream, workspace, workspace_bytes, log_probs_bf16, labels, xn, yn, costs, grads_bf16,
                          grad_scale, loss_sum, sync_counter, N, T, U, V, blank, fastemit_lambda, lse_mode, 1);
}

int rnnt_b200_rescale(void *stream, void *grads, const float *grad_out, int grad_out_stride, const float *applied,
                      int N, int64_t elems_per_sample, int elem_bytes) {
    if (N < 0 || elems_per_sample < 0 || grad_out_stride < 0 || grad_out_stride > 1 || !grads || !grad_out ||
        (elem_bytes != 4 && elem_bytes != 2))
        return RNNT_STATUS_INVALID_ARGUMENT;
    RNNT_TRY(launch_rescale((cudaStream_t)stream, grads, grad_out, grad_out_stride, applied, N, elems_per_sample,
                            elem_bytes == 2),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_loss_pairs(void *stream, void *workspace, size_t workspace_bytes, const float *pairs, const int *xn,
                         const int *yn, float *costs, float *pair_grads, int N, int T, int U,
                         float fastemit_lambda, int lse_mode) {
    if (!dense_args_ok(N, T, U, 2)) return RNNT_STATUS_INVALID_ARGUMENT;
    if ((reinterpret_cast<uintptr_t>(pairs) & 7u) || (reinterpret_cast<uintptr_t>(pair_grads) & 7u))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    FusedPlan plan;
    if (want_fused(N, T, U, &plan)) {
        RNNT_TRY(launch_fused(s, resolve_kind(lse_mode, false), plan, pairs, nullptr, xn, yn, costs, nullptr,
                              reinterpret_cast<float2 *>(pair_grads), nullptr, N, T, U, 2, 0, fastemit_lambda, 1, 1),
                 RNNT_STATUS_WARP_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    const Workspace w = carve(workspace, cells, N);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    const float2 *pr = reinterpret_cast<const float2 *>(pairs);
    RNNT_TRY(launch_wavefront(s, resolve_kind(lse_mode, false), p, pr, w.alphas, w.betas, w.ll, w.bad, costs,
                              pair_grads == nullptr, 1, T, U),
             RNNT_STATUS_WARP_FAILED);
    if (pair_grads)
        RNNT_TRY(launch_grads_pairs(s, p, pr, w.alphas, w.betas, w.bad, fastemit_lambda,
                                    reinterpret_cast<float2 *>(pair_grads), cells),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_gather_forward(void *stream, void *workspace, size_t workspace_bytes, const float *log_probs,
                             const int *labels, const int *xn, const int *yn, float *costs, float *pair_grads,
                             int N, int T, int U, int V, int blank, float fastemit_lambda, int lse_mode) {
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    FusedPlan plan;
    if (want_fused(N, T, U, &plan)) {
        RNNT_TRY(launch_fused(s, resolve_kind(lse_mode, false), plan, log_probs, labels, xn, yn, costs, nullptr,
                              reinterpret_cast<float2 *>(pair_grads), nullptr, N, T, U, V, blank, fastemit_lambda, 0, 1),
                 RNNT_STATUS_WARP_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    const Workspace w = carve(workspace, cells, N);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    RNNT_TRY(launch_gather(s, p, log_probs, labels, V, blank, w.pairs, nullptr, cells), RNNT_STATUS_GATHER_FAILED);
    RNNT_TRY(launch_wavefront(s, resolve_kind(lse_mode, false), p, w.pairs, w.alphas, w.betas, w.ll, w.bad, costs,
                              pair_grads == nullptr, 1, T, U),
             RNNT_STATUS_WARP_FAILED);
    if (pair_grads)
        RNNT_TRY(launch_grads_pairs(s, p, w.pairs, w.alphas, w.betas, w.bad, fastemit_lambda,
                                    reinterpret_cast<float2 *>(pair_grads), cells),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_logits_forward(void *stream, void *workspace, size_t workspace_bytes, const float *logits,
                              const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                              float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                              int lse_mode) {
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V || !lse) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    const Workspace w = carve(workspace, cells, N);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    // one pass over the logits: normaliser per cell + the two normalised log-probs the recurrence needs
    RNNT_TRY(launch_lse_pairs(s, logits, labels, N, T, U, V, blank, w.pairs, lse), RNNT_STATUS_GATHER_FAILED);
    // the (cells,2) layout from here on: same kernels as rnnt_b200_loss_pairs
    const int kind = resolve_kind(lse_mode, false);
    FusedPlan plan;
    if (want_fused(N, T, U, &plan)) {
        RNNT_TRY(launch_fused(s, kind, plan, reinterpret_cast<const float *>(w.pairs), nullptr, xn, yn, costs, nullptr,
                              reinterpret_cast<float2 *>(pair_grads), nullptr, N, T, U, 2, 0, fastemit_lambda, 1, 1),
                 RNNT_STATUS_WARP_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    RNNT_TRY(launch_wavefront(s, kind, p, w.pairs, w.alphas, w.betas, w.ll, w.bad, costs, pair_grads == nullptr, 1, T, U),
             RNNT_STATUS_WARP_FAILED);
    if (pair_grads)
        RNNT_TRY(launch_grads_pairs(s, p, w.pairs, w.alphas, w.betas, w.bad, fastemit_lambda,
                                    reinterpret_cast<float2 *>(pair_grads), cells),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_logits_backward(void *stream, const float *logits, const float *lse, const float *pair_grads,
                              const int *labels, const float *grad_out, float *out, int N, int T, int U, int V,
                              int blank) {
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    RNNT_TRY(launch_expand_logits((cudaStream_t)stream, logits, lse, reinterpret_cast<const float2 *>(pair_grads), labels,
                                  grad_out, out, N, T, U, V, blank),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_gather_backward(void *stream, const float *pair_grads, const int *labels, const float *grad_out,
                              float *out, int N, int T, int U, int V, int blank, int accumulate, const int *yn) {
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    Problem p = {nullptr, yn, nullptr, nullptr, N, T, U, 0};     // yn (optional): which labels are real
    ExpandSrc src = {};
    src.pg = reinterpret_cast<const float2 *>(pair_grads);
    src.scale = grad_out;
    src.labels = labels;
    src.label_adds = accumulate ? 1 : 0;
    RNNT_TRY(launch_expand((cudaStream_t)stream, p, src, out, (int64_t)N * T * U, V, blank),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_compact_forward(void *stream, void *workspace, size_t workspace_bytes, const float *xs, const int *ys,
                              const int *xn, const int *yn, float *costs, float *pair_grads, int64_t *loc,
                              int *totals, int64_t STU, int N, int V, int blank, float fastemit_lambda,
                              int lse_mode, int max_T, int max_U) {
    if (N < 0 || STU < 0 || V < 1 || V >= (1 << 22) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const Workspace w = carve(workspace, STU, N);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    RNNT_TRY(launch_prefix(s, xn, yn, N, w.mem_pref, w.lab_pref, totals ? totals : w.totals), RNNT_STATUS_GATHER_FAILED);
    Problem p = {xn, yn, w.mem_pref, w.lab_pref, N, 0, 0, 1};
    FusedPlan fplan;
    if (max_T > 0 && max_U > 0 && want_fused(N, max_T, max_U, &fplan)) {
        // small lattices: gather + wavefront + (cells,2) gradients + loc in one launch (no mismatch guard in the
        // compact reference, core_compact.cu:347-358)
        RNNT_TRY(launch_fused(s, resolve_kind(lse_mode, true), fplan, xs, ys, xn, yn, costs, nullptr,
                              reinterpret_cast<float2 *>(pair_grads), nullptr, N, max_T, max_U, V, blank,
                              fastemit_lambda, 0, 0, w.mem_pref, w.lab_pref, loc),
                 RNNT_STATUS_WARP_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    RNNT_TRY(launch_gather(s, p, xs, ys, V, blank, w.pairs, loc, STU), RNNT_STATUS_GATHER_FAILED);
    // no mismatch guard in the compact reference (core_compact.cu:347-358)
    RNNT_TRY(launch_wavefront(s, resolve_kind(lse_mode, true), p, w.pairs, w.alphas, w.betas, w.ll, w.bad, costs,
                              pair_grads == nullptr, 0, max_T, max_U),
             RNNT_STATUS_WARP_FAILED);
    if (pair_grads)
        RNNT_TRY(launch_grads_pairs(s, p, w.pairs, w.alphas, w.betas, nullptr, fastemit_lambda,
                                    reinterpret_cast<float2 *>(pair_grads), STU),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_compact_totals(void *stream, const int *xn, const int *yn, int N, int64_t *scratch, int *totals) {
    if (N <= 0 || !scratch || !totals) return RNNT_STATUS_INVALID_ARGUMENT;
    RNNT_TRY(launch_prefix((cudaStream_t)stream, xn, yn, N, scratch, scratch + N, totals), RNNT_STATUS_GATHER_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_joint_pack(void *stream, const float *f, const float *g, const int *lf, const int *lg, int64_t *scratch,
                         int *totals, float *x, int N, int T, int U1, int H, int64_t stu_hint) {
    if (N < 0 || T < 1 || U1 < 1 || H < 1 || !scratch) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    // mem_pref[n] = first packed row of lattice n: the same device prefix sums as the compact loss (lf = xn, lg = yn)
    RNNT_TRY(launch_prefix(s, lf, lg, N, scratch, scratch + N, totals), RNNT_STATUS_GATHER_FAILED);
    if (x) RNNT_TRY(launch_joint_pack(s, f, g, lf, lg, scratch, x, N, T, U1, H, stu_hint), RNNT_STATUS_GATHER_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_joint_pack_backward(void *stream, const float *dx, const int *lf, const int *lg, const int64_t *mem_pref,
                                  float *df, float *dg, int N, int T, int U1, int H) {
    if (N < 0 || T < 1 || U1 < 1 || H < 1 || !mem_pref || !dx) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    RNNT_TRY(launch_joint_grads((cudaStream_t)stream, dx, lf, lg, mem_pref, df, dg, N, T, U1, H),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_compact_backward(void *stream, const float *grad_cost, const float *pair_grads, const int64_t *loc,
                               const int *cum_lens, float *out, int64_t STU, int N, int V, int blank) {
    if (N < 0 || STU < 0 || V < 1 || V >= (1 << 22) || blank < 0 || blank >= V) return RNNT_STATUS_INVALID_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(pair_grads) & 7u) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0 || STU == 0) return RNNT_STATUS_SUCCESS;
    Problem p = {nullptr, nullptr, nullptr, nullptr, N, 0, 0, 1};
    ExpandSrc src = {};
    src.pg = reinterpret_cast<const float2 *>(pair_grads);
    src.scale = grad_cost;
    src.loc = loc;
    src.cum_lens = cum_lens;
    RNNT_TRY(launch_expand((cudaStream_t)stream, p, src, out, STU, V, blank), RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// ------------------------------------------------------------------------------------------
// (B) the reference's C ABI.  Scratch that the reference signatures have no room for comes
// from the stream-ordered allocator (cudaMallocAsync / cudaFreeAsync on the same stream).
// ------------------------------------------------------------------------------------------
static void compat_die(const char *what, int status) {
    // the reference's CHECK_KERNEL_STAT prints and exit(-1)s (core.h:7-14)
    fprintf(stderr, "%s error: %s\n", what, rnnt_b200_status_string(status));
    exit(-1);
}

int run_warp_rnnt(void *stream, unsigned int *counts, float *alphas, float *betas, const int *labels,
                  const float *log_probs, float *grads, float *costs, const int *xn, const int *yn, int N, int T,
                  int U, int V, int blank, float fastemit_lambda) {
    (void)counts;
    if (!dense_args_ok(N, T, U, V) || blank < 0 || blank >= V) return RNNT_STATUS_WARP_FAILED;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    const size_t pair_bytes = align_up((size_t)cells * sizeof(float2), 256);
    const size_t small = align_up(sizeof(float) * 2 * N, 256) + align_up(sizeof(int) * N, 256);
    char *tmp = nullptr;
    if (cudaMallocAsync((void **)&tmp, pair_bytes + small, s) != cudaSuccess) return RNNT_STATUS_WARP_FAILED;
    float2 *pairs = (float2 *)tmp;
    float *ll = (float *)(tmp + pair_bytes);
    int *bad = (int *)(tmp + pair_bytes + align_up(sizeof(float) * 2 * N, 256));
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    int status = RNNT_STATUS_SUCCESS;
    if (launch_gather(s, p, log_probs, labels, V, blank, pairs, nullptr, cells) != cudaSuccess)
        status = RNNT_STATUS_WARP_FAILED;
    if (!status && launch_wavefront(s, resolve_kind(RNNT_LSE_AUTO, false), p, pairs, alphas, betas, ll, bad, costs, 0,
                                    1, T, U) != cudaSuccess)
        status = RNNT_STATUS_WARP_FAILED;
    if (!status) {
        ExpandSrc src = {};
        src.pairs = pairs; src.alphas = alphas; src.betas = betas; src.bad = bad;
        src.labels = labels; src.fastemit_lambda = fastemit_lambda;
        if (launch_expand(s, p, src, grads, cells, V, blank) != cudaSuccess) status = RNNT_STATUS_GRADS_BLANK_FAILED;
    }
    cudaFreeAsync(tmp, s);
    return status;
}

int run_warp_rnnt_gather(void *stream, unsigned int *counts, float *alphas, float *betas, const float *log_probs,
                         float *grads, float *costs, const int *xn, const int *yn, int N, int T, int U,
                         float fastemit_lambda) {
    (void)counts;
    if (!dense_args_ok(N, T, U, 2)) return RNNT_STATUS_WARP_FAILED;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cells = (int64_t)N * T * U;
    const size_t llb = align_up(sizeof(float) * 2 * N, 256);
    char *tmp = nullptr;
    if (cudaMallocAsync((void **)&tmp, llb + align_up(sizeof(int) * N, 256), s) != cudaSuccess)
        return RNNT_STATUS_WARP_FAILED;
    float *ll = (float *)tmp;
    int *bad = (int *)(tmp + llb);
    Problem p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    const float2 *pr = reinterpret_cast<const float2 *>(log_probs);
    int status = RNNT_STATUS_SUCCESS;
    if (launch_wavefront(s, resolve_kind(RNNT_LSE_AUTO, false), p, pr, alphas, betas, ll, bad, costs, 0, 1, T, U) !=
        cudaSuccess)
        status = RNNT_STATUS_WARP_FAILED;
    if (!status && launch_grads_pairs(s, p, pr, alphas, betas, bad, fastemit_lambda, reinterpret_cast<float2 *>(grads),
                                      cells) != cudaSuccess)
        status = RNNT_STATUS_GRADS_BLANK_FAILED;
    cudaFreeAsync(tmp, s);
    return status;
}

// compact variants run on the legacy default stream like the reference (core.h:41-60 has no stream)
void run_gather_for_compact(const float *xs, const int *ys, const unsigned int *xn, const unsigned int *yn,
                            float *gather_xs, long *loc, const unsigned int *memPref, const unsigned int *labelPref,
                            unsigned int N, unsigned int T, unsigned int U, unsigned int V, unsigned int blank) {
    (void)memPref; (void)labelPref;   // recomputed on device in 64-bit
    if (N == 0) return;
    cudaStream_t s = 0;
    const size_t pb = align_up(sizeof(int64_t) * N, 256);
    char *tmp = nullptr;
    if (cudaMallocAsync((void **)&tmp, 2 * pb + 256, s) != cudaSuccess) compat_die("rnnt loss gather for compact", RNNT_STATUS_GATHER_FAILED);
    int64_t *mp = (int64_t *)tmp, *lp = (int64_t *)(tmp + pb);
    int *totals = (int *)(tmp + 2 * pb);
    const int *xi = (const int *)xn, *yi = (const int *)yn;
    bool ok = launch_prefix(s, xi, yi, (int)N, mp, lp, totals) == cudaSuccess;
    Problem p = {xi, yi, mp, lp, (int)N, 0, 0, 1};
    ok = ok && launch_gather(s, p, xs, ys, (int)V, (int)blank, reinterpret_cast<float2 *>(gather_xs),
                             reinterpret_cast<int64_t *>(loc), (int64_t)N * T * U) == cudaSuccess;
    cudaFreeAsync(tmp, s);
    if (!ok) compat_die("rnnt loss gather for compact", RNNT_STATUS_GATHER_FAILED);
}

void run_warp_rnnt_compact(unsigned int *counts, float *alphas, float *betas, const float *log_probs, float *grads,
                           float *costs, const unsigned int *xn, const unsigned int *yn, const unsigned int *memPref,
                           const unsigned int *labelPref, unsigned int N, unsigned int T, unsigned int U,
                           float fastemit_lambda, bool required_grad) {
    (void)counts; (void)memPref; (void)labelPref;
    if (N == 0) return;
    cudaStream_t s = 0;
    const size_t pb = align_up(sizeof(int64_t) * N, 256);
    const size_t llb = align_up(sizeof(float) * 2 * N, 256);
    char *tmp = nullptr;
    if (cudaMallocAsync((void **)&tmp, 2 * pb + llb + 256, s) != cudaSuccess) compat_die("rnnt loss compact betas", RNNT_STATUS_WARP_FAILED);
    int64_t *mp = (int64_t *)tmp, *lp = (int64_t *)(tmp + pb);
    float *ll = (float *)(tmp + 2 * pb);
    int *totals = (int *)(tmp + 2 * pb + llb);
    const int *xi = (const int *)xn, *yi = (const int *)yn;
    bool ok = launch_prefix(s, xi, yi, (int)N, mp, lp, totals) == cudaSuccess;
    Problem p = {xi, yi, mp, lp, (int)N, 0, 0, 1};
    const float2 *pr = reinterpret_cast<const float2 *>(log_probs);
    ok = ok && launch_wavefront(s, resolve_kind(RNNT_LSE_AUTO, true), p, pr, alphas, betas, ll, nullptr, costs,
                                required_grad ? 0 : 1, 0, (int)T, (int)U) == cudaSuccess;
    if (ok && required_grad)
        ok = launch_grads_pairs(s, p, pr, alphas, betas, nullptr, fastemit_lambda, reinterpret_cast<float2 *>(grads),
                                (int64_t)N * T * U) == cudaSuccess;
    cudaFreeAsync(tmp, s);
    if (!ok) compat_die("rnnt loss compact", RNNT_STATUS_WARP_FAILED);
}

void run_scatter_grad_for_compact(const float *grad_cost, const float *gather_grad, const long *loc,
                                  const int *cum_lens, float *scatter_grad, unsigned int STU, unsigned int N,
                                  unsigned int V, unsigned int blank) {
    const int st = rnnt_b200_compact_backward(nullptr, grad_cost, gather_grad, reinterpret_cast<const int64_t *>(loc),
                                              cum_lens, scatter_grad, (int64_t)STU, (int)N, (int)V, (int)blank);
    if (st != RNNT_STATUS_SUCCESS) compat_die("rnnt loss filling scatter grad", st);
}

}  // extern "C"
