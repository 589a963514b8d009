// api.cu -- the extern "C" surface of librnnt_b200.so (declared in include/rnnt_b200.h).
//
// (A) rnnt_b200_*: native interface bound by csrc/binding.cpp.
// (B) run_warp_rnnt & co: the reference's C ABI (the reference's core.h:29-60) implemented on top
//     of (A)'s kernels so the reference's own bindings link against this library unchanged.
#include <atomic>
#include <cmath>
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

// per thread, so that calls from several host threads (one per device) neither race nor see each other's launches
static thread_local int32_t t_record[RNNT_LAUNCH_RECORD_LEN];
static thread_local int32_t t_record_seq;
int32_t *launch_record() { return t_record; }
void begin_launch_record(int path) {
    memset(t_record, 0, sizeof(t_record));
    t_record[RNNT_REC_SEQ] = ++t_record_seq;
    t_record[RNNT_REC_PATH] = path;
    t_record[RNNT_REC_GROUPS] = 1;
}

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
// full-size test bounds it at 2.5e-4).  The exact chain is ~2x longer per anti-diagonal; on an H100 (700 W) the dense
// cfg-2 call's gradient write follows the recurrence (composed emit, fused.cu), so the recurrence is on its critical
// path: the timeline (tools/fused_timeline.py) shows beta[0,0] at ~51 us exact and ~46 us fast, of a ~80 us kernel.
// RNNT_LSE_FAST / RNNT_B200_LSE=fast selects the short chain.
static bool fast_lse(int lse_mode) {
    if (lse_mode == RNNT_LSE_AUTO) lse_mode = default_lse_mode();
    return lse_mode == RNNT_LSE_FAST;
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

static bool dense_args_ok(int N, int T, int U, int V, int blank) {
    if (N < 0 || T < 1 || U < 1 || V < 1) return false;
    if ((int64_t)T * U >= (int64_t)1 << 31) return false;
    if ((int64_t)N * T * U >= (int64_t)1 << 31) return false;   // cell ids are 32-bit in the emit kernel
    if (V >= (1 << 22)) return false;
    return blank >= 0 && blank < V;
}
static bool compact_args_ok(int N, int64_t STU, int V, int blank) {
    return N >= 0 && STU >= 0 && V >= 1 && V < (1 << 22) && blank >= 0 && blank < V;
}
// pruned (N,T,S,V) window rows over a full (N,T,U) lattice: the full lattice as dense_args_ok takes it, and row ids
// that fit 32 bits as cell ids do
static bool pruned_args_ok(int N, int T, int S, int U, int V, int blank) {
    return S >= 1 && dense_args_ok(N, T, U, V, blank) && (int64_t)N * T * S < (int64_t)1 << 31;
}
// the simple loss: the (N,T,U) lattice as dense_args_ok takes it; its contractions put N on the grid's z axis
static bool simple_args_ok(int N, int T, int U, int V, int blank) {
    return dense_args_ok(N, T, U, V, blank) && N <= 65535;
}
// the simple loss's saved buffer: norm (N,T,U), then the row offsets of am (N,T) and of lm (N,U)
static SimpleArgs simple_call(const float *am, const float *lm, const int *labels, const int *xn, const int *yn,
                              float *saved, int N, int T, int U, int V, int blank) {
    SimpleArgs a = {};
    a.am = am; a.lm = lm; a.labels = labels; a.xn = xn; a.yn = yn;
    a.norm = saved;
    a.off_a = saved + (int64_t)N * T * U;
    a.off_l = a.off_a + (int64_t)N * T;
    a.T = T; a.U = U; a.V = V; a.blank = blank;
    return a;
}
// k2's smoothing scales: finite, >= 0, sl + sa < 1 (so c = 1 - sl - sa > 0)
static bool smooth_scales_ok(float sl, float sa) {
    return std::isfinite(sl) && std::isfinite(sa) && sl >= 0.0f && sa >= 0.0f && (double)sl + (double)sa < 1.0;
}
static bool smoothed(float sl, float sa) { return sl > 0.0f || sa > 0.0f; }
// the smoothed loss's saved buffer: the simple loss's, then Ll (N,U), Am (N,T), log uni (V)
static int64_t simple_saved_len(int N, int T, int U, int V, bool smooth) {
    const int64_t n = N, base = n * T * U + n * T + n * U;
    return smooth ? base + n * U + n * T + V : base;
}
// the smoothed workspace: forward = the loss's, then uni (V) and the unigram partials; backward = c*grad_out (N),
// Cb, Cl (N,U), the G partials and G (V); one size covers both
struct SmoothWorkspace {
    float *uni, *upart, *cgo, *cb, *cl, *gpart, *G;
    size_t fwd_bytes, bwd_bytes;
};
static SmoothWorkspace carve_smooth(void *base, int N, int T, int U, int V) {
    SmoothWorkspace w;
    const size_t n = (size_t)max(N, 0), t = (size_t)max(T, 0), u = (size_t)max(U, 0), v = (size_t)max(V, 0);
    size_t off = carve(nullptr, (int64_t)(n * t * u), N).bytes;
    auto take = [&](size_t bytes) {
        void *p = base ? (void *)((char *)base + off) : nullptr;
        off += align_up(bytes, 256);
        return (float *)p;
    };
    w.uni = take(v * sizeof(float));
    w.upart = take((n * u + kSmoothRows - 1) / kSmoothRows * v * sizeof(float));
    w.fwd_bytes = off;
    off = 0;
    w.cgo = take(n * sizeof(float));
    w.cb = take(n * u * sizeof(float));
    w.cl = take(n * u * sizeof(float));
    w.gpart = take((n * t + kSmoothRows - 1) / kSmoothRows * v * sizeof(float));
    w.G = take(v * sizeof(float));
    w.bwd_bytes = off;
    return w;
}
static SmoothArgs smooth_call(const SimpleArgs &a, const SmoothWorkspace &w, float *saved, int N, float sl, float sa) {
    SmoothArgs m = {};
    m.am = a.am; m.lm = a.lm; m.labels = a.labels; m.xn = a.xn; m.yn = a.yn;
    m.off_a = a.off_a; m.off_l = a.off_l;
    m.Ll = saved + simple_saved_len(N, a.T, a.U, a.V, false);
    m.Am = m.Ll + (int64_t)N * a.U;
    m.loguni = m.Am + (int64_t)N * a.T;
    m.uni = w.uni; m.upart = w.upart;
    m.cgo = w.cgo; m.cb = w.cb; m.cl = w.cl; m.gpart = w.gpart; m.G = w.G;
    m.c = (float)(1.0 - (double)sl - (double)sa);
    m.sl = sl; m.sa = sa;
    m.N = N; m.T = a.T; m.U = a.U; m.V = a.V; m.blank = a.blank;
    return m;
}
// (cells,2) pairs and their gradients are read and written as float2
static bool pairs_aligned(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
// k_fill_pairs writes the workspace's pairs, carved at its base, two cells per float4
static bool workspace_aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

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

// One loss call, described on the host; run_loss runs it.
struct LossCall {
    Problem p;                   // dense (N,T,U), or compact with its device prefix sums (p.T = p.U = 0)
    int T, U;                    // lattice bounds: p.T, p.U (dense); max_T, max_U (compact; 0 = unknown)
    int64_t cells;               // N*T*U (dense) or STU (compact)
    // source: log-probs of V elements per cell (f32 or bf16) with their labels, or ready-made (cells,2) pairs
    const void *lp;
    const int *labels;
    int V, blank, io_bf16;
    const float2 *pairs;
    // outputs: costs, plus the dense gradient (with scale and the reduced loss), or the (cells,2) gradient, or neither
    float *costs;
    void *grads;
    const float *grad_scale;
    float *loss_sum;
    unsigned *sync_counter;      // with loss_sum: reduce in the fused kernel, else in a launch of its own
    float2 *pair_grads;
    int64_t *loc;                // compact gather: label id per cell, or null
    float fastemit_lambda;
    int lse_mode;
};

static LossCall dense_call(const int *xn, const int *yn, int N, int T, int U, float *costs, float fastemit_lambda,
                           int lse_mode) {
    LossCall c = {};
    c.p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    c.T = T; c.U = U; c.cells = (int64_t)N * T * U;
    c.costs = costs; c.fastemit_lambda = fastemit_lambda; c.lse_mode = lse_mode;
    return c;
}

static LossCall compact_call(const int *xn, const int *yn, const int64_t *mem_pref, const int64_t *lab_pref, int N,
                             int64_t STU, int max_T, int max_U, float *costs, float fastemit_lambda, int lse_mode) {
    LossCall c = {};
    c.p = {xn, yn, mem_pref, lab_pref, N, 0, 0, 1};
    c.T = max_T; c.U = max_U; c.cells = STU;
    c.costs = costs; c.fastemit_lambda = fastemit_lambda; c.lse_mode = lse_mode;
    return c;
}

// the workspace carved for a call on `cells` cells; false when the caller's is missing or too small
static bool carve_ok(void *workspace, size_t workspace_bytes, int64_t cells, int N, Workspace *w) {
    *w = carve(workspace, cells, N);
    return workspace && workspace_bytes >= w->bytes;
}

// Large batches of large lattices: software-pipeline lattice groups over internal streams so that the
// latency-bound wavefront of group g overlaps the bandwidth-bound gather of g+1 and emit of g-1.
// ... which only pays when the wavefront (a per-lattice latency chain of T+U-1 steps that does not shrink with the
// group) is short against the bandwidth-bound emit: cfg 5's micro-batch takes the pipeline, cfg 4 does not.
// The two estimates (0.45 us per anti-diagonal, an emit at 5.5 TB/s) were measured on a B200 and have not been
// re-derived for the H100 (3.35 TB/s HBM3): there the emit is slower, so the true break-even favours the pipeline more often than this estimate.
static int pipeline_groups(const LossCall &c) {
    const int N = c.p.N;
    const double wave_us = 0.45 * (c.T + c.U), emit_us = (double)c.cells * c.V * (c.io_bf16 ? 2 : 4) / 5.5e6;
    return (c.grads && N >= 8 && (int64_t)c.cells * c.V * 4 >= ((int64_t)512 << 20) && pipeline_enabled() &&
            wave_us < 0.4 * emit_us)
               ? (N >= 32 ? 8 : 4) : 1;
}

// the general path of a dense call with dense gradients, one lattice group after another over the pipeline's streams
static int run_pipelined(cudaStream_t s, Pipeline *pl, const LossCall &c, const Workspace &w, int groups) {
    const int N = c.p.N, T = c.T, U = c.U, V = c.V;
    const size_t esz = c.io_bf16 ? 2 : 4;
    const bool fast = fast_lse(c.lse_mode);
    int status = RNNT_STATUS_SUCCESS;
    cudaEventRecord(pl->fork, s);
    cudaStreamWaitEvent(pl->gather_s, pl->fork, 0);
    cudaStreamWaitEvent(pl->expand_s, pl->fork, 0);
    for (int i = 0; i < Pipeline::kWave; ++i) cudaStreamWaitEvent(pl->wave_s[i], pl->fork, 0);
    for (int g = 0; g < groups && !status; ++g) {
        const int n0 = (int)((int64_t)N * g / groups), n1 = (int)((int64_t)N * (g + 1) / groups);
        const int ng = n1 - n0;
        const int64_t c0 = (int64_t)n0 * T * U, cg = (int64_t)ng * T * U;
        Problem p = {c.p.xn + n0, c.p.yn + n0, nullptr, nullptr, ng, T, U, 0};
        const int *lab_g = c.labels + (int64_t)n0 * (U - 1);
        const void *lp_g = (const char *)c.lp + (size_t)c0 * V * esz;
        void *grads_g = (char *)c.grads + (size_t)c0 * V * esz;
        cudaStream_t ws = pl->wave_s[g % Pipeline::kWave];
        if (launch_gather(pl->gather_s, p, lp_g, lab_g, V, c.blank, w.pairs + c0, nullptr, cg, c.io_bf16) != cudaSuccess)
            status = RNNT_STATUS_GATHER_FAILED;
        cudaEventRecord(pl->gathered[g], pl->gather_s);
        cudaStreamWaitEvent(ws, pl->gathered[g], 0);
        if (!status && launch_wavefront(ws, fast, p, w.pairs + c0, w.alphas + c0, w.betas + c0, w.ll + 2 * n0,
                                        w.bad + n0, c.costs + n0, 0, T, U) != cudaSuccess)
            status = RNNT_STATUS_WARP_FAILED;
        cudaEventRecord(pl->swept[g], ws);
        cudaStreamWaitEvent(pl->expand_s, pl->swept[g], 0);
        ExpandSrc src = {};
        src.pairs = w.pairs + c0; src.alphas = w.alphas + c0; src.betas = w.betas + c0; src.bad = w.bad + n0;
        src.scale = c.grad_scale ? c.grad_scale + n0 : nullptr; src.labels = lab_g;
        src.fastemit_lambda = c.fastemit_lambda;
        if (!status && launch_expand(pl->expand_s, p, src, grads_g, cg, V, c.blank, true, c.io_bf16) != cudaSuccess)
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
    if (!status && c.loss_sum && launch_loss_sum(s, c.costs, c.grad_scale, N, c.loss_sum) != cudaSuccess)
        status = RNNT_STATUS_COSTS_FAILED;
    return status;
}

// Runs one loss call (N > 0, arguments checked): the fused kernel when the lattices fit it, else the general path --
// gather (unless the pairs are given), wavefront, then the dense emit or the (cells,2) gradients.  Only the general
// path needs the workspace.
static int run_loss(cudaStream_t s, void *workspace, size_t workspace_bytes, const LossCall &c) {
    const Problem &p = c.p;
    FusedPlan plan;
    if (c.T > 0 && c.U > 0 && want_fused(p.N, c.T, c.U, &plan)) {
        FusedCall f = {};
        f.fast_lse = fast_lse(c.lse_mode);
        if (c.pairs) {
            f.lp = c.pairs; f.V = 2; f.pairs_in = 1;
        } else {
            f.lp = c.lp; f.labels = c.labels; f.V = c.V; f.blank = c.blank; f.io_bf16 = c.io_bf16;
        }
        f.xn = p.xn; f.yn = p.yn; f.mem_pref = p.mem_pref; f.lab_pref = p.lab_pref; f.loc = c.loc;
        f.costs = c.costs; f.grads = c.grads; f.pair_grads = c.pair_grads; f.scale = c.grad_scale;
        f.loss_sum = c.loss_sum; f.sync_counter = c.sync_counter;
        f.N = p.N; f.T = c.T; f.U = c.U; f.lam = c.fastemit_lambda;
        RNNT_TRY(launch_fused(s, plan, f), RNNT_STATUS_WARP_FAILED);
        if (c.loss_sum && !c.sync_counter)                  // no counter: reduce in a second, tiny launch
            RNNT_TRY(launch_loss_sum(s, c.costs, c.grad_scale, p.N, c.loss_sum), RNNT_STATUS_COSTS_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, c.cells, p.N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    const int groups = pipeline_groups(c);
    if (groups > 1) {
        std::lock_guard<std::mutex> lock(g_pipe_mu);    // the pipeline's events are shared by all calls on this device
        if (Pipeline *pl = get_pipeline_locked()) {
            const int status = run_pipelined(s, pl, c, w, groups);
            launch_record()[RNNT_REC_GROUPS] = groups;
            return status;
        }
    }
    const bool fast = fast_lse(c.lse_mode);
    const float2 *pairs = c.pairs;
    if (!pairs) {
        RNNT_TRY(launch_gather(s, p, c.lp, c.labels, c.V, c.blank, w.pairs, c.loc, c.cells, c.io_bf16),
                 RNNT_STATUS_GATHER_FAILED);
        pairs = w.pairs;
    }
    RNNT_TRY(launch_wavefront(s, fast, p, pairs, w.alphas, w.betas, w.ll, w.bad, c.costs, !c.grads && !c.pair_grads,
                              c.T, c.U),
             RNNT_STATUS_WARP_FAILED);
    if (c.grads) {
        ExpandSrc src = {};
        src.pairs = pairs; src.alphas = w.alphas; src.betas = w.betas; src.bad = w.bad;
        src.scale = c.grad_scale; src.labels = c.labels; src.fastemit_lambda = c.fastemit_lambda;
        RNNT_TRY(launch_expand(s, p, src, c.grads, c.cells, c.V, c.blank, false, c.io_bf16),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    }
    if (c.pair_grads)
        RNNT_TRY(launch_grads_pairs(s, p, pairs, w.alphas, w.betas, p.compact ? nullptr : w.bad, c.fastemit_lambda,
                                    c.pair_grads, c.cells),
                 RNNT_STATUS_GRADS_BLANK_FAILED);
    if (c.loss_sum) RNNT_TRY(launch_loss_sum(s, c.costs, c.grad_scale, p.N, c.loss_sum), RNNT_STATUS_COSTS_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// k2's lattice type and delay penalty (include/rnnt_b200.h): 0 regular, 1 modified, 2 constrained; lam finite, >= 0.
// The one-symbol-per-frame types take no FastEmit and rows of at most kFramesMaxU columns.
static bool path_type_ok(int rnnt_type, float delay_penalty, float fastemit_lambda, int U) {
    if (rnnt_type < 0 || rnnt_type > 2 || !std::isfinite(delay_penalty) || delay_penalty < 0.0f) return false;
    return rnnt_type == 0 || (fastemit_lambda == 0.0f && U <= kFramesMaxU);
}

// A dense k2-family call on its pairs c.pairs (the workspace's, or the caller's): the delay penalty into the workspace's
// pairs, then the regular driver (run_loss) or the frame sweep.  raw_blank: k_frames_grads' unfolded blank slots, or null.
static int run_typed(cudaStream_t s, void *workspace, size_t workspace_bytes, const Workspace &w, LossCall c,
                     int rnnt_type, float delay_penalty, float *raw_blank) {
    const bool delayed = delay_penalty != 0.0f;
    if (delayed) {
        RNNT_TRY(launch_delay_pairs(s, c.pairs, w.pairs, c.p.xn, c.p.yn, c.p.N, c.T, c.U, delay_penalty),
                 RNNT_STATUS_GATHER_FAILED);
        c.pairs = w.pairs;
    }
    if (rnnt_type == 0) return run_loss(s, workspace, workspace_bytes, c);
    FramesCall f = {};
    f.pairs = c.pairs; f.xn = c.p.xn; f.yn = c.p.yn;
    f.alphas = w.alphas; f.betas = w.betas; f.ll = w.ll; f.status = w.bad;
    f.costs = c.costs; f.pair_grads = c.pair_grads; f.raw_blank = c.pair_grads ? raw_blank : nullptr;
    f.N = c.p.N; f.T = c.T; f.U = c.U; f.constrained = rnnt_type == 2;
    RNNT_TRY(launch_frames(s, f, delayed), RNNT_STATUS_WARP_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// dense layout, log_probs / grads of 4-byte (f32) or 2-byte (bf16) elements
static int loss_dense_any(void *stream, void *workspace, size_t workspace_bytes, const void *log_probs,
                          const int *labels, const int *xn, const int *yn, float *costs, void *grads,
                          const float *grad_scale, float *loss_sum, unsigned int *sync_counter, int N, int T,
                          int U, int V, int blank, float fastemit_lambda, int lse_mode, int io_bf16) {
    if ((io_bf16 && !grads) || !dense_args_ok(N, T, U, V, blank)) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    LossCall c = dense_call(xn, yn, N, T, U, costs, fastemit_lambda, lse_mode);
    c.lp = log_probs; c.labels = labels; c.V = V; c.blank = blank; c.io_bf16 = io_bf16;
    c.grads = grads; c.grad_scale = grad_scale; c.loss_sum = loss_sum; c.sync_counter = sync_counter;
    return run_loss((cudaStream_t)stream, workspace, workspace_bytes, c);
}

// the HAT normalisation needs a label column besides the blank
static bool hat_ok(int hat, int V) { return !hat || V >= 2; }

// a 4-byte (f32) or 2-byte (bf16) element size, and p aligned to it
static bool elem_ok(const void *p, int elem_bytes) {
    return (elem_bytes == 4 || elem_bytes == 2) && !(reinterpret_cast<uintptr_t>(p) & (uintptr_t)(elem_bytes - 1));
}

// loss from logits of 4-byte (f32) or 2-byte (bf16) elements: the normaliser pass reads them, the recurrence and
// everything after it run on the f32 (cells,2) pairs and do not see the element type (nor the normalisation: hat)
static int logits_forward_any(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                              const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                              float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                              int lse_mode, int io_bf16, int rnnt_type, float delay_penalty, int hat = 0) {
    if (!dense_args_ok(N, T, U, V, blank) || !lse || !pairs_aligned(pair_grads) ||
        !path_type_ok(rnnt_type, delay_penalty, fastemit_lambda, U) || !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    LossCall c = dense_call(xn, yn, N, T, U, costs, fastemit_lambda, lse_mode);
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, c.cells, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    // one pass over the logits: normaliser per cell + the two normalised log-probs the recurrence needs
    RNNT_TRY(launch_lse_pairs(s, logits, labels, N, T, U, V, blank, w.pairs, lse, io_bf16, hat),
             RNNT_STATUS_GATHER_FAILED);
    c.pairs = w.pairs; c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_typed(s, workspace, workspace_bytes, w, c, rnnt_type, delay_penalty, nullptr);
}

static int logits_backward_any(void *stream, const void *logits, const float *lse, const float *pair_grads,
                               const int *labels, const float *grad_out, void *out, int N, int T, int U, int V,
                               int blank, int io_bf16, int hat = 0) {
    if (!dense_args_ok(N, T, U, V, blank) || !pairs_aligned(pair_grads) || !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    RNNT_TRY(launch_expand_logits((cudaStream_t)stream, logits, lse, reinterpret_cast<const float2 *>(pair_grads), labels,
                                  grad_out, out, N, T, U, V, blank, io_bf16, hat),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// compact (STU,V) logits in joint_pack's row order: the normaliser pass over the ragged rows, then the recurrence of
// rnnt_b200_compact_forward on the (STU,2) pairs
static int logits_compact_forward_any(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                      const int *ys, const int *xn, const int *yn, float *costs, float *lse,
                                      float *pair_grads, int64_t *prefix, int *totals, int64_t STU, int N, int V,
                                      int blank, float fastemit_lambda, int lse_mode, int max_T, int max_U,
                                      int io_bf16, int hat = 0) {
    if (!compact_args_ok(N, STU, V, blank) || !lse || !prefix || !pairs_aligned(pair_grads) || !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, STU, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    RNNT_TRY(launch_prefix(s, xn, yn, N, prefix, prefix + N, totals ? totals : w.totals), RNNT_STATUS_GATHER_FAILED);
    LossCall c = compact_call(xn, yn, prefix, prefix + N, N, STU, max_T, max_U, costs, fastemit_lambda, lse_mode);
    RNNT_TRY(launch_lse_pairs_compact(s, logits, c.p, ys, STU, V, blank, w.pairs, lse, io_bf16, hat),
             RNNT_STATUS_GATHER_FAILED);
    c.pairs = w.pairs; c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_loss(s, workspace, workspace_bytes, c);
}

// One alignment call (rnnt_b200_align_*): compact prefix sums, the gather into (cells,2) pairs, then k_align -- the
// max-plus alpha sweep and the backtrace in one launch.
struct AlignCall {
    Problem p;                   // dense (N,T,U); compact: p.compact = 1, its prefix sums come from the workspace
    int T, U;                    // lattice bounds: dense p.T, p.U; compact max_T, max_U (both > 0)
    int64_t cells;               // N*T*U (dense) or STU (compact)
    const void *lp;
    const int *labels;
    int V, blank, io_bf16;
    int hat;                     // alignment from logits: the HAT normalisation instead of log_softmax
    float *scores;
    int *frames;
};

struct AlignWorkspace {
    float2 *pairs;
    float *alphas;
    uint32_t *dec;
    int64_t *mem_pref, *lab_pref;
    int *totals;
    size_t bytes;
};

static AlignWorkspace carve_align(void *base, int64_t cells, int N, int T, int U) {
    AlignWorkspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void *p = base ? (void *)((char *)base + off) : nullptr;
        off += align_up(bytes, 256);
        return p;
    };
    const size_t c = (size_t)(cells > 0 ? cells : 0), n = (size_t)(N > 0 ? N : 0);
    const size_t words = n * (size_t)((max(U, 0) + 31) / 32) * (size_t)(max(T, 0) + 31);
    w.pairs = (float2 *)take(c * sizeof(float2));
    w.alphas = (float *)take(c * sizeof(float));
    w.dec = (uint32_t *)take(words * sizeof(uint32_t));
    w.mem_pref = (int64_t *)take(n * sizeof(int64_t));
    w.lab_pref = (int64_t *)take(n * sizeof(int64_t));
    w.totals = (int *)take(4 * sizeof(int));
    w.bytes = off;
    return w;
}

static int run_align(cudaStream_t s, void *workspace, size_t workspace_bytes, AlignCall c) {
    const AlignWorkspace w = carve_align(workspace, c.cells, c.p.N, c.T, c.U);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    if (c.p.compact) {
        RNNT_TRY(launch_prefix(s, c.p.xn, c.p.yn, c.p.N, w.mem_pref, w.lab_pref, w.totals), RNNT_STATUS_GATHER_FAILED);
        c.p.mem_pref = w.mem_pref;
        c.p.lab_pref = w.lab_pref;
    }
    RNNT_TRY(launch_gather(s, c.p, c.lp, c.labels, c.V, c.blank, w.pairs, nullptr, c.cells, c.io_bf16),
             RNNT_STATUS_GATHER_FAILED);
    RNNT_TRY(launch_align(s, c.p, w.pairs, w.alphas, w.dec, c.T, c.U, c.scores, c.frames), RNNT_STATUS_WARP_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// The alignment from logits (rnnt_b200_align_logits_*): run_align's workspace, then the normaliser's lse (cells).  Its
// decision words (N, ceil(U/32), T+31) also hold k_frames_align's (N, ceil(U/32), T).
static size_t align_logits_bytes(int64_t cells, int N, int T, int U) {
    return carve_align(nullptr, cells, N, T, U).bytes + align_up((size_t)(cells > 0 ? cells : 0) * sizeof(float), 256);
}

// compact prefix sums, the normaliser pass into the workspace's pairs and lse, the delay penalty in place, then k_align
// (regular) or k_frames_align (modified, constrained); c.lp holds the logits
static int run_align_logits(cudaStream_t s, void *workspace, size_t workspace_bytes, AlignCall c, int rnnt_type,
                            float delay_penalty) {
    if (!workspace || workspace_bytes < align_logits_bytes(c.cells, c.p.N, c.T, c.U))
        return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    const AlignWorkspace w = carve_align(workspace, c.cells, c.p.N, c.T, c.U);
    float *lse = reinterpret_cast<float *>(static_cast<char *>(workspace) + w.bytes);
    if (c.p.compact) {
        RNNT_TRY(launch_prefix(s, c.p.xn, c.p.yn, c.p.N, w.mem_pref, w.lab_pref, w.totals), RNNT_STATUS_GATHER_FAILED);
        c.p.mem_pref = w.mem_pref;
        c.p.lab_pref = w.lab_pref;
        RNNT_TRY(launch_lse_pairs_compact(s, c.lp, c.p, c.labels, c.cells, c.V, c.blank, w.pairs, lse, c.io_bf16,
                                          c.hat),
                 RNNT_STATUS_GATHER_FAILED);
    } else {
        RNNT_TRY(launch_lse_pairs(s, c.lp, c.labels, c.p.N, c.T, c.U, c.V, c.blank, w.pairs, lse, c.io_bf16, c.hat),
                 RNNT_STATUS_GATHER_FAILED);
    }
    if (delay_penalty != 0.0f)
        RNNT_TRY(launch_delay_pairs(s, w.pairs, w.pairs, c.p.xn, c.p.yn, c.p.N, c.T, c.U, delay_penalty),
                 RNNT_STATUS_GATHER_FAILED);
    if (rnnt_type == 0) {
        RNNT_TRY(launch_align(s, c.p, w.pairs, w.alphas, w.dec, c.T, c.U, c.scores, c.frames), RNNT_STATUS_WARP_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    FramesAlignCall f = {};
    f.pairs = w.pairs; f.xn = c.p.xn; f.yn = c.p.yn; f.dec = w.dec; f.scores = c.scores; f.frames = c.frames;
    f.N = c.p.N; f.T = c.T; f.U = c.U; f.constrained = rnnt_type == 2; f.delayed = delay_penalty != 0.0f;
    RNNT_TRY(launch_frames_align(s, f), RNNT_STATUS_WARP_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// the alignment from dense (N,T,U,V) logits of 4- or 2-byte elements (hat: the HAT normalisation)
static int align_logits_dense_any(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                  const int *labels, const int *xn, const int *yn, float *scores, int *frames, int N,
                                  int T, int U, int V, int blank, int elem_bytes, int rnnt_type, float delay_penalty,
                                  int hat) {
    if (!elem_ok(logits, elem_bytes) || !dense_args_ok(N, T, U, V, blank) || !hat_ok(hat, V) ||
        !path_type_ok(rnnt_type, delay_penalty, 0.0f, U) || !scores || !frames || !workspace_aligned16(workspace))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    AlignCall c = {};
    c.p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    c.T = T; c.U = U; c.cells = (int64_t)N * T * U;
    c.lp = logits; c.labels = labels; c.V = V; c.blank = blank; c.io_bf16 = elem_bytes == 2; c.hat = hat;
    c.scores = scores; c.frames = frames;
    return run_align_logits((cudaStream_t)stream, workspace, workspace_bytes, c, rnnt_type, delay_penalty);
}

// ... and from compact (STU,V) logits in joint_pack's row order (regular lattice, no penalty)
static int align_logits_compact_any(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                    const int *labels, const int *xn, const int *yn, float *scores, int *frames,
                                    int64_t STU, int N, int V, int blank, int elem_bytes, int max_T, int max_U,
                                    int hat) {
    if (!elem_ok(logits, elem_bytes) || !compact_args_ok(N, STU, V, blank) || !hat_ok(hat, V) || max_T <= 0 ||
        max_U <= 0 || !scores || !frames || !workspace_aligned16(workspace))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    AlignCall c = {};
    c.p = {xn, yn, nullptr, nullptr, N, 0, 0, 1};
    c.T = max_T; c.U = max_U; c.cells = STU;
    c.lp = logits; c.labels = labels; c.V = V; c.blank = blank; c.io_bf16 = elem_bytes == 2; c.hat = hat;
    c.scores = scores; c.frames = frames;
    return run_align_logits((cudaStream_t)stream, workspace, workspace_bytes, c, 0, 0.0f);
}

static int logits_compact_backward_any(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                       const int *ys, const int *xn, const int *yn, const int64_t *prefix,
                                       const float *grad_out, void *out, int64_t STU, int N, int V, int blank,
                                       int io_bf16, int hat = 0) {
    if (!compact_args_ok(N, STU, V, blank) || !lse || !prefix || !pairs_aligned(pair_grads) || !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0 || STU == 0) return RNNT_STATUS_SUCCESS;
    const Problem p = {xn, yn, prefix, prefix + N, N, 0, 0, 1};
    RNNT_TRY(launch_expand_logits_compact((cudaStream_t)stream, logits, lse, reinterpret_cast<const float2 *>(pair_grads),
                                          p, ys, grad_out, out, STU, V, blank, io_bf16, hat),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// rnnt_loss_pruned's (N,T,S,V) window rows of 4- or 2-byte elements on the full (N,T,U) lattice
static int logits_pruned_forward_any(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                     const int *labels, const int *xn, const int *yn, const int *ranges, float *costs,
                                     float *lse, float *pair_grads, int N, int T, int S, int U, int V,
                                     int blank, float fastemit_lambda, int lse_mode, int elem_bytes, int rnnt_type,
                                     float delay_penalty, int hat) {
    if (!elem_ok(logits, elem_bytes) || !pruned_args_ok(N, T, S, U, V, blank) || !lse || !pairs_aligned(pair_grads) ||
        !workspace_aligned16(workspace) || !path_type_ok(rnnt_type, delay_penalty, fastemit_lambda, U) ||
        !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    LossCall c = dense_call(xn, yn, N, T, U, costs, fastemit_lambda, lse_mode);
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, c.cells, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    // one pass over the window rows: their normalisers, and the full lattice's pairs ((kBig, kBig) off the windows)
    RNNT_TRY(launch_lse_pairs_pruned(s, logits, labels, ranges, N, T, S, U, V, blank, w.pairs, lse, elem_bytes == 2,
                                     hat),
             RNNT_STATUS_GATHER_FAILED);
    c.pairs = w.pairs; c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_typed(s, workspace, workspace_bytes, w, c, rnnt_type, delay_penalty, nullptr);
}

static int logits_pruned_backward_any(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                      const int *labels, const int *ranges, const float *grad_out, void *out, int N,
                                      int T, int S, int U, int V, int blank, int elem_bytes, int hat) {
    if (!elem_ok(logits, elem_bytes) || !elem_ok(out, elem_bytes) || !pruned_args_ok(N, T, S, U, V, blank) ||
        !pairs_aligned(pair_grads) || !hat_ok(hat, V))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    RNNT_TRY(launch_expand_logits_pruned((cudaStream_t)stream, logits, lse, reinterpret_cast<const float2 *>(pair_grads),
                                         labels, ranges, grad_out, out, N, T, S, U, V, blank, elem_bytes == 2, hat),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// TDT: its own entry points (a cell carries 2 + D values, not the pair run_loss drives).  durations: strictly
// increasing, in [0, 16], at least one > 0.
static bool tdt_durations(const int *durations, int D, TdtDurations *out) {
    if (!durations || D < 1 || D > kTdtMaxD) return false;
    *out = {};
    out->D = D;
    for (int j = 0; j < D; ++j) {
        const int d = durations[j];
        if (d < 0 || d > 16 || (j > 0 && d <= durations[j - 1])) return false;
        out->d[j] = d;
    }
    out->dmax = durations[D - 1];
    return out->dmax > 0;
}
// Multi-blank: B big blanks with durations strictly increasing in [2, 16] (so B <= 15), in the durations' place
static bool mb_durations(const int *durations, int B, TdtDurations *out) {
    if (!durations || B < 1 || B > kTdtMaxD - 2) return false;
    *out = {};
    out->D = B;
    for (int j = 0; j < B; ++j) {
        const int d = durations[j];
        if (d < 2 || d > 16 || (j > 0 && d <= durations[j - 1])) return false;
        out->d[j] = d;
    }
    out->dmax = durations[B - 1];
    return true;
}
// The arguments every TDT or multi-blank call (mb) takes, dense or compact: the family's durations into dur, the
// logits' element size and alignment, the row and the blank, sigma finite and >= 0, then the layout's sizes.  A TDT row
// is V token logits then D duration logits, blank in [0, V); a multi-blank row is V logits, the standard blank at
// `blank` and big blank i at blank - 1 - i, so blank in [B, V).  Dense: T, U >= 1 and N*T*U < 2^31; compact: STU < 2^31
// in place of N*T*U, and N <= 65535 (the normaliser's grid holds one CTA row per lattice).
static bool tdt_args_ok(bool mb, bool compact, const int *durations, int D, float sigma, int N, int64_t STU, int T,
                        int U, int V, int blank, int elem_bytes, const void *logits, TdtDurations *dur) {
    return (mb ? mb_durations(durations, D, dur) : tdt_durations(durations, D, dur)) && elem_ok(logits, elem_bytes) &&
           V >= 1 && (int64_t)V + (mb ? 0 : D) < ((int64_t)1 << 22) && blank >= (mb ? D : 0) && blank < V &&
           std::isfinite(sigma) && sigma >= 0.0f && N >= 0 &&
           (compact ? N <= 65535 && STU >= 0 && STU < ((int64_t)1 << 31)
                    : T >= 1 && U >= 1 && (int64_t)N * T * U < ((int64_t)1 << 31));
}
// cells: N*T*U (dense) or STU (compact); the compact call also takes 4 ints for the totals it does not return
struct TdtWorkspace { float *lp, *alpha, *beta, *ll; int *status, *totals; size_t bytes; };
static TdtWorkspace carve_tdt(void *base, int64_t cells, int N, int D, bool compact) {
    TdtWorkspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void *p = base ? (void *)((char *)base + off) : nullptr;
        off += align_up(bytes, 256);
        return p;
    };
    const size_t c = (size_t)max(cells, (int64_t)0), n = (size_t)max(N, 0);
    w.lp = (float *)take(c * (size_t)(2 + max(D, 0)) * sizeof(float));
    w.alpha = (float *)take(c * sizeof(float));
    w.beta = (float *)take(c * sizeof(float));
    w.ll = (float *)take(n * sizeof(float));
    w.status = (int *)take(n * sizeof(int));
    w.totals = compact ? (int *)take(4 * sizeof(int)) : nullptr;
    w.bytes = off;
    return w;
}
// The TDT alignment (rnnt_b200_tdt_align_*), one size for both layouts: lse (cells,2), lp (cells,2+D), alpha (cells),
// the decision bytes (cells), status (N), then the compact call's prefix sums (2N) and totals (4).
struct TdtAlignWorkspace {
    float2 *lse;
    float *lp, *alpha;
    uint8_t *dec;
    int *status;
    int64_t *prefix;
    int *totals;
    size_t bytes;
};
static TdtAlignWorkspace carve_tdt_align(void *base, int64_t cells, int N, int D) {
    TdtAlignWorkspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void *p = base ? (void *)((char *)base + off) : nullptr;
        off += align_up(bytes, 256);
        return p;
    };
    const size_t c = (size_t)max(cells, (int64_t)0), n = (size_t)max(N, 0);
    w.lse = (float2 *)take(c * sizeof(float2));
    w.lp = (float *)take(c * (size_t)(2 + max(D, 0)) * sizeof(float));
    w.alpha = (float *)take(c * sizeof(float));
    w.dec = (uint8_t *)take(c);
    w.status = (int *)take(n * sizeof(int));
    w.prefix = (int64_t *)take(2 * n * sizeof(int64_t));
    w.totals = (int *)take(4 * sizeof(int));
    w.bytes = off;
    return w;
}

// The TDT and multi-blank calls (mb), dense (N,T,U) or compact (STU rows, T and U the bounds max_T, max_U).  Nothing
// is launched before a refusal: the arguments first, then the N == 0 return, then the workspace.  The TDT lse is
// (cells,2) (lse_tok, lse_dur) pairs, read and written as float2; the multi-blank lse is one float per cell.

// the loss: the compact prefix sums into prefix (and totals, or the workspace's), then launch_tdt_forward
static int tdt_forward_any(bool mb, bool compact, void *stream, void *workspace, size_t workspace_bytes,
                           const void *logits, const int *labels, const int *xn, const int *yn, const int *durations,
                           int D, float sigma, float *costs, float *lse, float *grads, int64_t *prefix, int *totals,
                           int64_t STU, int N, int T, int U, int V, int blank, int elem_bytes) {
    TdtDurations dur;
    if (!tdt_args_ok(mb, compact, durations, D, sigma, N, STU, T, U, V, blank, elem_bytes, logits, &dur) || !costs ||
        !lse || (!mb && !pairs_aligned(lse)) || !workspace_aligned16(workspace) ||
        (compact && (!prefix || T < 1 || U < 1)))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    const TdtWorkspace w = carve_tdt(workspace, compact ? STU : (int64_t)N * T * U, N, D, compact);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    cudaStream_t s = (cudaStream_t)stream;
    TdtFwd c = {};
    if (compact) {
        RNNT_TRY(launch_prefix(s, xn, yn, N, prefix, prefix + N, totals ? totals : w.totals),
                 RNNT_STATUS_GATHER_FAILED);
        c.mem_pref = prefix; c.lab_pref = prefix + N; c.STU = STU;
    }
    c.x = logits; c.labels = labels; c.xn = xn; c.yn = yn; c.costs = costs; c.pg = grads;
    c.lp = w.lp; c.alpha = w.alpha; c.beta = w.beta; c.ll = w.ll; c.status = w.status;
    c.N = N; c.T = T; c.U = U; c.V = V; c.blank = blank; c.sigma = sigma; c.dur = dur; c.io_bf16 = elem_bytes == 2;
    c.multiblank = mb;
    if (mb) c.lse_mb = lse; else c.lse = reinterpret_cast<float2 *>(lse);
    RNNT_TRY(launch_tdt_forward(s, c), RNNT_STATUS_WARP_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// the gradient (T, U: 0 when compact; yn and prefix: compact only)
static int tdt_backward_any(bool mb, bool compact, void *stream, const void *logits, const float *lse,
                            const float *grads, const int *labels, const int *yn, const int *durations, int D,
                            const int64_t *prefix, const float *grad_out, void *out, int64_t STU, int N, int T, int U,
                            int V, int blank, int elem_bytes) {
    TdtDurations dur;
    if (!tdt_args_ok(mb, compact, durations, D, 0.0f, N, STU, T, U, V, blank, elem_bytes, logits, &dur) ||
        !elem_ok(out, elem_bytes) || !lse || (!mb && !pairs_aligned(lse)) || !grads || !out || (compact && !prefix))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0 || (compact && STU == 0)) return RNNT_STATUS_SUCCESS;
    TdtBwd c = {};
    if (compact) {
        c.yn = yn; c.mem_pref = prefix; c.lab_pref = prefix + N; c.STU = STU;
    }
    c.x = logits; c.pg = grads; c.labels = labels; c.grad_out = grad_out; c.out = out;
    c.N = N; c.T = T; c.U = U; c.V = V; c.D = D; c.blank = blank; c.io_bf16 = elem_bytes == 2;
    c.multiblank = mb;
    if (mb) c.lse_mb = lse; else c.lse = reinterpret_cast<const float2 *>(lse);
    RNNT_TRY(launch_tdt_backward((cudaStream_t)stream, c), RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

// the Viterbi alignment: the compact prefix sums into the workspace, then launch_tdt_align, whose third output is
// the label durations, or launch_mb_align, whose third output is the blank counts
static int tdt_align_any(bool mb, bool compact, void *stream, void *workspace, size_t workspace_bytes,
                         const void *logits, const int *labels, const int *xn, const int *yn, const int *durations,
                         int D, float sigma, float *scores, int *frames, int *third, int64_t STU, int N, int T, int U,
                         int V, int blank, int elem_bytes) {
    TdtDurations dur;
    if (!tdt_args_ok(mb, compact, durations, D, sigma, N, STU, T, U, V, blank, elem_bytes, logits, &dur) || !scores ||
        !frames || !third || !workspace_aligned16(workspace) || (compact && (T < 1 || U < 1)))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    const TdtAlignWorkspace w = carve_tdt_align(workspace, compact ? STU : (int64_t)N * T * U, N, D);
    if (!workspace || workspace_bytes < w.bytes) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    cudaStream_t s = (cudaStream_t)stream;
    TdtFwd c = {};
    if (compact) {
        RNNT_TRY(launch_prefix(s, xn, yn, N, w.prefix, w.prefix + N, w.totals), RNNT_STATUS_GATHER_FAILED);
        c.mem_pref = w.prefix; c.lab_pref = w.prefix + N; c.STU = STU;
    }
    c.x = logits; c.labels = labels; c.xn = xn; c.yn = yn; c.costs = scores;
    c.lp = w.lp; c.alpha = w.alpha; c.status = w.status;
    c.N = N; c.T = T; c.U = U; c.V = V; c.blank = blank; c.sigma = sigma; c.dur = dur; c.io_bf16 = elem_bytes == 2;
    c.multiblank = mb;
    if (mb) c.lse_mb = (float *)w.lse; else c.lse = w.lse;
    const auto align = mb ? launch_mb_align : launch_tdt_align;
    RNNT_TRY(align(s, c, w.dec, frames, third), RNNT_STATUS_WARP_FAILED);
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
void rnnt_b200_debug_last_launch(int32_t *out) {
    if (out) memcpy(out, rnnt::launch_record(), sizeof(int32_t) * RNNT_LAUNCH_RECORD_LEN);
}

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
    return rnnt_b200_loss_pairs_ex(stream, workspace, workspace_bytes, pairs, xn, yn, costs, pair_grads, N, T, U,
                                   fastemit_lambda, lse_mode, 0, 0.0f);
}

int rnnt_b200_loss_pairs_ex(void *stream, void *workspace, size_t workspace_bytes, const float *pairs, const int *xn,
                            const int *yn, float *costs, float *pair_grads, int N, int T, int U, float fastemit_lambda,
                            int lse_mode, int rnnt_type, float delay_penalty) {
    if (!dense_args_ok(N, T, U, 2, 0) || !pairs_aligned(pairs) || !pairs_aligned(pair_grads) ||
        !path_type_ok(rnnt_type, delay_penalty, fastemit_lambda, U))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    LossCall c = dense_call(xn, yn, N, T, U, costs, fastemit_lambda, lse_mode);
    c.pairs = reinterpret_cast<const float2 *>(pairs); c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    if (rnnt_type == 0 && delay_penalty == 0.0f)        // the regular loss: the fused kernel needs no workspace
        return run_loss((cudaStream_t)stream, workspace, workspace_bytes, c);
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, c.cells, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    return run_typed((cudaStream_t)stream, workspace, workspace_bytes, w, c, rnnt_type, delay_penalty, nullptr);
}

int rnnt_b200_gather_forward(void *stream, void *workspace, size_t workspace_bytes, const float *log_probs,
                             const int *labels, const int *xn, const int *yn, float *costs, float *pair_grads,
                             int N, int T, int U, int V, int blank, float fastemit_lambda, int lse_mode) {
    if (!dense_args_ok(N, T, U, V, blank) || !pairs_aligned(pair_grads)) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    LossCall c = dense_call(xn, yn, N, T, U, costs, fastemit_lambda, lse_mode);
    c.lp = log_probs; c.labels = labels; c.V = V; c.blank = blank; c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_loss((cudaStream_t)stream, workspace, workspace_bytes, c);
}

int rnnt_b200_logits_forward(void *stream, void *workspace, size_t workspace_bytes, const float *logits,
                              const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                              float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                              int lse_mode) {
    return rnnt_b200_logits_forward_ex(stream, workspace, workspace_bytes, logits, labels, xn, yn, costs, lse,
                                       pair_grads, N, T, U, V, blank, fastemit_lambda, lse_mode, 0, 0.0f);
}

int rnnt_b200_logits_forward_ex(void *stream, void *workspace, size_t workspace_bytes, const float *logits,
                                const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                                float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                                int lse_mode, int rnnt_type, float delay_penalty) {
    return logits_forward_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, costs, lse, pair_grads, N, T,
                              U, V, blank, fastemit_lambda, lse_mode, 0, rnnt_type, delay_penalty);
}

int rnnt_b200_logits_backward(void *stream, const float *logits, const float *lse, const float *pair_grads,
                              const int *labels, const float *grad_out, float *out, int N, int T, int U, int V,
                              int blank) {
    return logits_backward_any(stream, logits, lse, pair_grads, labels, grad_out, out, N, T, U, V, blank, 0);
}

int rnnt_b200_logits_forward_bf16(void *stream, void *workspace, size_t workspace_bytes, const void *logits_bf16,
                                  const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                                  float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                                  int lse_mode) {
    return rnnt_b200_logits_forward_bf16_ex(stream, workspace, workspace_bytes, logits_bf16, labels, xn, yn, costs, lse,
                                            pair_grads, N, T, U, V, blank, fastemit_lambda, lse_mode, 0, 0.0f);
}

int rnnt_b200_logits_forward_bf16_ex(void *stream, void *workspace, size_t workspace_bytes, const void *logits_bf16,
                                     const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                                     float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                                     int lse_mode, int rnnt_type, float delay_penalty) {
    if (reinterpret_cast<uintptr_t>(logits_bf16) & 1u) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_forward_any(stream, workspace, workspace_bytes, logits_bf16, labels, xn, yn, costs, lse, pair_grads,
                              N, T, U, V, blank, fastemit_lambda, lse_mode, 1, rnnt_type, delay_penalty);
}

int rnnt_b200_logits_backward_bf16(void *stream, const void *logits_bf16, const float *lse, const float *pair_grads,
                                   const int *labels, const float *grad_out, void *out_bf16, int N, int T, int U, int V,
                                   int blank) {
    if ((reinterpret_cast<uintptr_t>(logits_bf16) | reinterpret_cast<uintptr_t>(out_bf16)) & 1u)
        return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_backward_any(stream, logits_bf16, lse, pair_grads, labels, grad_out, out_bf16, N, T, U, V, blank, 1);
}

int rnnt_b200_gather_backward(void *stream, const float *pair_grads, const int *labels, const float *grad_out,
                              float *out, int N, int T, int U, int V, int blank, int accumulate, const int *yn) {
    if (!dense_args_ok(N, T, U, V, blank) || !pairs_aligned(pair_grads)) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    Problem p = {nullptr, yn, nullptr, nullptr, N, T, U, 0};     // yn (optional): which labels are real
    ExpandSrc src = {};
    src.pg = reinterpret_cast<const float2 *>(pair_grads);
    src.scale = grad_out;
    src.labels = labels;
    src.label_adds = accumulate ? 1 : 0;
    RNNT_TRY(launch_expand((cudaStream_t)stream, p, src, out, (int64_t)N * T * U, V, blank, false, 0),
             RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_compact_forward(void *stream, void *workspace, size_t workspace_bytes, const float *xs, const int *ys,
                              const int *xn, const int *yn, float *costs, float *pair_grads, int64_t *loc,
                              int *totals, int64_t STU, int N, int V, int blank, float fastemit_lambda,
                              int lse_mode, int max_T, int max_U) {
    if (!compact_args_ok(N, STU, V, blank) || !pairs_aligned(pair_grads)) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    cudaStream_t s = (cudaStream_t)stream;
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, STU, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    RNNT_TRY(launch_prefix(s, xn, yn, N, w.mem_pref, w.lab_pref, totals ? totals : w.totals), RNNT_STATUS_GATHER_FAILED);
    LossCall c = compact_call(xn, yn, w.mem_pref, w.lab_pref, N, STU, max_T, max_U, costs, fastemit_lambda, lse_mode);
    c.lp = xs; c.labels = ys; c.V = V; c.blank = blank; c.loc = loc;
    c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_loss(s, workspace, workspace_bytes, c);
}

int rnnt_b200_logits_compact_forward(void *stream, void *workspace, size_t workspace_bytes, const float *logits,
                                     const int *ys, const int *xn, const int *yn, float *costs, float *lse,
                                     float *pair_grads, int64_t *prefix, int *totals, int64_t STU, int N, int V,
                                     int blank, float fastemit_lambda, int lse_mode, int max_T, int max_U) {
    return logits_compact_forward_any(stream, workspace, workspace_bytes, logits, ys, xn, yn, costs, lse, pair_grads,
                                      prefix, totals, STU, N, V, blank, fastemit_lambda, lse_mode, max_T, max_U, 0);
}

int rnnt_b200_logits_compact_forward_bf16(void *stream, void *workspace, size_t workspace_bytes,
                                          const void *logits_bf16, const int *ys, const int *xn, const int *yn,
                                          float *costs, float *lse, float *pair_grads, int64_t *prefix, int *totals,
                                          int64_t STU, int N, int V, int blank, float fastemit_lambda, int lse_mode,
                                          int max_T, int max_U) {
    if (reinterpret_cast<uintptr_t>(logits_bf16) & 1u) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_compact_forward_any(stream, workspace, workspace_bytes, logits_bf16, ys, xn, yn, costs, lse,
                                      pair_grads, prefix, totals, STU, N, V, blank, fastemit_lambda, lse_mode, max_T,
                                      max_U, 1);
}

int rnnt_b200_logits_compact_backward(void *stream, const float *logits, const float *lse, const float *pair_grads,
                                      const int *ys, const int *xn, const int *yn, const int64_t *prefix,
                                      const float *grad_out, float *out, int64_t STU, int N, int V, int blank) {
    return logits_compact_backward_any(stream, logits, lse, pair_grads, ys, xn, yn, prefix, grad_out, out, STU, N, V,
                                       blank, 0);
}

int rnnt_b200_logits_compact_backward_bf16(void *stream, const void *logits_bf16, const float *lse,
                                           const float *pair_grads, const int *ys, const int *xn, const int *yn,
                                           const int64_t *prefix, const float *grad_out, void *out_bf16, int64_t STU,
                                           int N, int V, int blank) {
    if ((reinterpret_cast<uintptr_t>(logits_bf16) | reinterpret_cast<uintptr_t>(out_bf16)) & 1u)
        return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_compact_backward_any(stream, logits_bf16, lse, pair_grads, ys, xn, yn, prefix, grad_out, out_bf16,
                                       STU, N, V, blank, 1);
}

int rnnt_b200_logits_pruned_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                    const int *labels, const int *xn, const int *yn, const int *ranges, float *costs,
                                    float *lse, float *pair_grads, int N, int T, int S, int U, int V, int blank,
                                    float fastemit_lambda, int lse_mode, int elem_bytes) {
    return rnnt_b200_logits_pruned_forward_ex(stream, workspace, workspace_bytes, logits, labels, xn, yn, ranges, costs,
                                              lse, pair_grads, N, T, S, U, V, blank, fastemit_lambda, lse_mode,
                                              elem_bytes, 0, 0.0f);
}

int rnnt_b200_logits_pruned_forward_ex(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                       const int *labels, const int *xn, const int *yn, const int *ranges,
                                       float *costs, float *lse, float *pair_grads, int N, int T, int S, int U, int V,
                                       int blank, float fastemit_lambda, int lse_mode, int elem_bytes, int rnnt_type,
                                       float delay_penalty) {
    return logits_pruned_forward_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, ranges, costs, lse,
                                     pair_grads, N, T, S, U, V, blank, fastemit_lambda, lse_mode, elem_bytes,
                                     rnnt_type, delay_penalty, 0);
}

int rnnt_b200_logits_pruned_backward(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                     const int *labels, const int *ranges, const float *grad_out, void *out, int N,
                                     int T, int S, int U, int V, int blank, int elem_bytes) {
    return logits_pruned_backward_any(stream, logits, lse, pair_grads, labels, ranges, grad_out, out, N, T, S, U, V,
                                      blank, elem_bytes, 0);
}

// HAT twins of the from-logits entries: the same drivers and workspaces, the HAT normalisation in the logits passes

int rnnt_b200_logits_hat_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                 const int *labels, const int *xn, const int *yn, float *costs, float *lse,
                                 float *pair_grads, int N, int T, int U, int V, int blank, float fastemit_lambda,
                                 int lse_mode, int elem_bytes, int rnnt_type, float delay_penalty) {
    if (!elem_ok(logits, elem_bytes)) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_forward_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, costs, lse, pair_grads, N, T,
                              U, V, blank, fastemit_lambda, lse_mode, elem_bytes == 2, rnnt_type, delay_penalty, 1);
}

int rnnt_b200_logits_hat_backward(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                  const int *labels, const float *grad_out, void *out, int N, int T, int U, int V,
                                  int blank, int elem_bytes) {
    if (!elem_ok(logits, elem_bytes) || !elem_ok(out, elem_bytes)) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_backward_any(stream, logits, lse, pair_grads, labels, grad_out, out, N, T, U, V, blank,
                               elem_bytes == 2, 1);
}

int rnnt_b200_logits_compact_hat_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                         const int *ys, const int *xn, const int *yn, float *costs, float *lse,
                                         float *pair_grads, int64_t *prefix, int *totals, int64_t STU, int N, int V,
                                         int blank, float fastemit_lambda, int lse_mode, int max_T, int max_U,
                                         int elem_bytes) {
    if (!elem_ok(logits, elem_bytes)) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_compact_forward_any(stream, workspace, workspace_bytes, logits, ys, xn, yn, costs, lse, pair_grads,
                                      prefix, totals, STU, N, V, blank, fastemit_lambda, lse_mode, max_T, max_U,
                                      elem_bytes == 2, 1);
}

int rnnt_b200_logits_compact_hat_backward(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                          const int *ys, const int *xn, const int *yn, const int64_t *prefix,
                                          const float *grad_out, void *out, int64_t STU, int N, int V, int blank,
                                          int elem_bytes) {
    if (!elem_ok(logits, elem_bytes) || !elem_ok(out, elem_bytes)) return RNNT_STATUS_INVALID_ARGUMENT;
    return logits_compact_backward_any(stream, logits, lse, pair_grads, ys, xn, yn, prefix, grad_out, out, STU, N, V,
                                       blank, elem_bytes == 2, 1);
}

int rnnt_b200_logits_pruned_hat_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                        const int *labels, const int *xn, const int *yn, const int *ranges,
                                        float *costs, float *lse, float *pair_grads, int N, int T, int S, int U, int V,
                                        int blank, float fastemit_lambda, int lse_mode, int elem_bytes, int rnnt_type,
                                        float delay_penalty) {
    return logits_pruned_forward_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, ranges, costs, lse,
                                     pair_grads, N, T, S, U, V, blank, fastemit_lambda, lse_mode, elem_bytes,
                                     rnnt_type, delay_penalty, 1);
}

int rnnt_b200_logits_pruned_hat_backward(void *stream, const void *logits, const float *lse, const float *pair_grads,
                                         const int *labels, const int *ranges, const float *grad_out, void *out, int N,
                                         int T, int S, int U, int V, int blank, int elem_bytes) {
    return logits_pruned_backward_any(stream, logits, lse, pair_grads, labels, ranges, grad_out, out, N, T, S, U, V,
                                      blank, elem_bytes, 1);
}

size_t rnnt_b200_tdt_workspace_bytes(int N, int T, int U, int num_durations) {
    return carve_tdt(nullptr, (int64_t)max(N, 0) * max(T, 0) * max(U, 0), N, num_durations, false).bytes;
}

int rnnt_b200_tdt_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits, const int *labels,
                          const int *xn, const int *yn, const int *durations, int num_durations, float sigma,
                          float *costs, float *lse, float *grads, int N, int T, int U, int V, int blank,
                          int elem_bytes) {
    return tdt_forward_any(false, false, stream, workspace, workspace_bytes, logits, labels, xn, yn, durations,
                           num_durations, sigma, costs, lse, grads, nullptr, nullptr, 0, N, T, U, V, blank,
                           elem_bytes);
}

int rnnt_b200_tdt_backward(void *stream, const void *logits, const float *lse, const float *grads, const int *labels,
                           const int *durations, int num_durations, const float *grad_out, void *out, int N, int T,
                           int U, int V, int blank, int elem_bytes) {
    return tdt_backward_any(false, false, stream, logits, lse, grads, labels, nullptr, durations, num_durations,
                            nullptr, grad_out, out, 0, N, T, U, V, blank, elem_bytes);
}

size_t rnnt_b200_tdt_compact_workspace_bytes(int64_t STU, int N, int num_durations) {
    return carve_tdt(nullptr, STU, N, num_durations, true).bytes;
}

int rnnt_b200_tdt_compact_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                  const int *labels, const int *xn, const int *yn, const int *durations,
                                  int num_durations, float sigma, float *costs, float *lse, float *grads,
                                  int64_t *prefix, int *totals, int64_t STU, int N, int V, int blank, int elem_bytes,
                                  int max_T, int max_U) {
    return tdt_forward_any(false, true, stream, workspace, workspace_bytes, logits, labels, xn, yn, durations,
                           num_durations, sigma, costs, lse, grads, prefix, totals, STU, N, max_T, max_U, V, blank,
                           elem_bytes);
}

int rnnt_b200_tdt_compact_backward(void *stream, const void *logits, const float *lse, const float *grads,
                                   const int *labels, const int *yn, const int *durations, int num_durations,
                                   const int64_t *prefix, const float *grad_out, void *out, int64_t STU, int N, int V,
                                   int blank, int elem_bytes) {
    return tdt_backward_any(false, true, stream, logits, lse, grads, labels, yn, durations, num_durations, prefix,
                            grad_out, out, STU, N, 0, 0, V, blank, elem_bytes);
}

size_t rnnt_b200_tdt_align_workspace_bytes(int64_t cells, int N, int num_durations) {
    return carve_tdt_align(nullptr, cells, N, num_durations).bytes;
}

int rnnt_b200_tdt_align_dense(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                              const int *labels, const int *xn, const int *yn, const int *durations, int num_durations,
                              float sigma, float *scores, int *frames, int *label_durations, int N, int T, int U,
                              int V, int blank, int elem_bytes) {
    return tdt_align_any(false, false, stream, workspace, workspace_bytes, logits, labels, xn, yn, durations,
                         num_durations, sigma, scores, frames, label_durations, 0, N, T, U, V, blank, elem_bytes);
}

int rnnt_b200_tdt_align_compact(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                const int *labels, const int *xn, const int *yn, const int *durations,
                                int num_durations, float sigma, float *scores, int *frames, int *label_durations,
                                int64_t STU, int N, int V, int blank, int elem_bytes, int max_T, int max_U) {
    return tdt_align_any(false, true, stream, workspace, workspace_bytes, logits, labels, xn, yn, durations,
                         num_durations, sigma, scores, frames, label_durations, STU, N, max_T, max_U, V, blank,
                         elem_bytes);
}

// The multi-blank alignment carves the TDT alignment's workspace with D = B; its lse is one float per cell, held in
// the first half of the lse slot.
size_t rnnt_b200_multiblank_align_workspace_bytes(int64_t cells, int N, int num_big_blanks) {
    return rnnt_b200_tdt_align_workspace_bytes(cells, N, num_big_blanks);
}

int rnnt_b200_multiblank_align_dense(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                     const int *labels, const int *xn, const int *yn, const int *big_blank_durations,
                                     int num_big_blanks, float sigma, float *scores, int *frames, int *blank_counts,
                                     int N, int T, int U, int V, int blank, int elem_bytes) {
    return tdt_align_any(true, false, stream, workspace, workspace_bytes, logits, labels, xn, yn, big_blank_durations,
                         num_big_blanks, sigma, scores, frames, blank_counts, 0, N, T, U, V, blank, elem_bytes);
}

int rnnt_b200_multiblank_align_compact(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                       const int *labels, const int *xn, const int *yn,
                                       const int *big_blank_durations, int num_big_blanks, float sigma, float *scores,
                                       int *frames, int *blank_counts, int64_t STU, int N, int V, int blank,
                                       int elem_bytes, int max_T, int max_U) {
    return tdt_align_any(true, true, stream, workspace, workspace_bytes, logits, labels, xn, yn, big_blank_durations,
                         num_big_blanks, sigma, scores, frames, blank_counts, STU, N, max_T, max_U, V, blank,
                         elem_bytes);
}

size_t rnnt_b200_multiblank_workspace_bytes(int N, int T, int U, int num_big_blanks) {
    return rnnt_b200_tdt_workspace_bytes(N, T, U, num_big_blanks);
}

int rnnt_b200_multiblank_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                 const int *labels, const int *xn, const int *yn, const int *big_blank_durations,
                                 int num_big_blanks, float sigma, float *costs, float *lse, float *grads, int N, int T,
                                 int U, int V, int blank, int elem_bytes) {
    return tdt_forward_any(true, false, stream, workspace, workspace_bytes, logits, labels, xn, yn,
                           big_blank_durations, num_big_blanks, sigma, costs, lse, grads, nullptr, nullptr, 0, N, T, U,
                           V, blank, elem_bytes);
}

int rnnt_b200_multiblank_backward(void *stream, const void *logits, const float *lse, const float *grads,
                                  const int *labels, const int *big_blank_durations, int num_big_blanks,
                                  const float *grad_out, void *out, int N, int T, int U, int V, int blank,
                                  int elem_bytes) {
    return tdt_backward_any(true, false, stream, logits, lse, grads, labels, nullptr, big_blank_durations,
                            num_big_blanks, nullptr, grad_out, out, 0, N, T, U, V, blank, elem_bytes);
}

size_t rnnt_b200_multiblank_compact_workspace_bytes(int64_t STU, int N, int num_big_blanks) {
    return rnnt_b200_tdt_compact_workspace_bytes(STU, N, num_big_blanks);
}

int rnnt_b200_multiblank_compact_forward(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                         const int *labels, const int *xn, const int *yn,
                                         const int *big_blank_durations, int num_big_blanks, float sigma,
                                         float *costs, float *lse, float *grads, int64_t *prefix, int *totals,
                                         int64_t STU, int N, int V, int blank, int elem_bytes, int max_T, int max_U) {
    return tdt_forward_any(true, true, stream, workspace, workspace_bytes, logits, labels, xn, yn,
                           big_blank_durations, num_big_blanks, sigma, costs, lse, grads, prefix, totals, STU, N,
                           max_T, max_U, V, blank, elem_bytes);
}

int rnnt_b200_multiblank_compact_backward(void *stream, const void *logits, const float *lse, const float *grads,
                                          const int *labels, const int *yn, const int *big_blank_durations,
                                          int num_big_blanks, const int64_t *prefix, const float *grad_out, void *out,
                                          int64_t STU, int N, int V, int blank, int elem_bytes) {
    return tdt_backward_any(true, true, stream, logits, lse, grads, labels, yn, big_blank_durations, num_big_blanks,
                            prefix, grad_out, out, STU, N, 0, 0, V, blank, elem_bytes);
}

void rnnt_b200_debug_last_tdt_launch(int32_t *out) {
    if (out) rnnt::tdt_launch_record(out);
}

void rnnt_b200_debug_last_frames_launch(int32_t *out) {
    if (out) rnnt::frames_launch_record(out);
}

void rnnt_b200_debug_last_frames_align_launch(int32_t *out) {
    if (out) rnnt::frames_align_launch_record(out);
}

size_t rnnt_b200_simple_workspace_bytes(int N, int T, int U) {
    return carve(nullptr, (int64_t)max(N, 0) * max(T, 0) * max(U, 0), N).bytes;
}

size_t rnnt_b200_simple_smoothed_workspace_bytes(int N, int T, int U, int V) {
    const SmoothWorkspace w = carve_smooth(nullptr, N, T, U, V);
    return max(w.fwd_bytes, w.bwd_bytes);
}

int rnnt_b200_simple_forward(void *stream, void *workspace, size_t workspace_bytes, const float *am, const float *lm,
                             const int *labels, const int *xn, const int *yn, float *costs, float *saved,
                             float *pair_grads, int N, int T, int U, int V, int blank, int lse_mode) {
    return rnnt_b200_simple_smoothed_forward(stream, workspace, workspace_bytes, am, lm, labels, xn, yn, costs, saved,
                                             pair_grads, N, T, U, V, blank, lse_mode, 0.0f, 0.0f);
}

int rnnt_b200_simple_backward(void *stream, const float *am, const float *lm, const int *labels, const int *xn,
                              const int *yn, const float *saved, const float *pair_grads, const float *grad_out,
                              float *dam, float *dlm, int N, int T, int U, int V, int blank) {
    return rnnt_b200_simple_smoothed_backward(stream, nullptr, 0, am, lm, labels, xn, yn, saved, pair_grads, grad_out,
                                              dam, dlm, N, T, U, V, blank, 0.0f, 0.0f);
}

int rnnt_b200_simple_smoothed_forward(void *stream, void *workspace, size_t workspace_bytes, const float *am,
                                      const float *lm, const int *labels, const int *xn, const int *yn, float *costs,
                                      float *saved, float *pair_grads, int N, int T, int U, int V, int blank,
                                      int lse_mode, float lm_only_scale, float am_only_scale) {
    return rnnt_b200_simple_smoothed_forward_ex(stream, workspace, workspace_bytes, am, lm, labels, xn, yn, costs, saved,
                                                pair_grads, N, T, U, V, blank, lse_mode, lm_only_scale, am_only_scale,
                                                0, 0.0f, nullptr);
}

int rnnt_b200_simple_smoothed_forward_ex(void *stream, void *workspace, size_t workspace_bytes, const float *am,
                                         const float *lm, const int *labels, const int *xn, const int *yn,
                                         float *costs, float *saved, float *pair_grads, int N, int T, int U, int V,
                                         int blank, int lse_mode, float lm_only_scale, float am_only_scale,
                                         int rnnt_type, float delay_penalty, float *raw_blank_grads) {
    if (!simple_args_ok(N, T, U, V, blank) || !smooth_scales_ok(lm_only_scale, am_only_scale) || !saved ||
        !pairs_aligned(pair_grads) || !pairs_aligned(workspace) ||
        !path_type_ok(rnnt_type, delay_penalty, 0.0f, U) || (raw_blank_grads && !pair_grads))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    const bool smooth = smoothed(lm_only_scale, am_only_scale);
    cudaStream_t s = (cudaStream_t)stream;
    LossCall c = dense_call(xn, yn, N, T, U, costs, 0.0f, lse_mode);
    Workspace w;
    if (!carve_ok(workspace, workspace_bytes, c.cells, N, &w)) return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    if (smooth && workspace_bytes < rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, V))
        return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    SimpleArgs a = simple_call(am, lm, labels, xn, yn, saved, N, T, U, V, blank);
    a.pairs = w.pairs;
    RNNT_TRY(launch_simple_forward(s, a, N), RNNT_STATUS_GATHER_FAILED);
    if (smooth) {
        SmoothArgs m = smooth_call(a, carve_smooth(workspace, N, T, U, V), saved, N, lm_only_scale, am_only_scale);
        m.pairs = w.pairs;
        // with sa = 0 nothing computes Am and log uni: they are saved as 0
        if (!(am_only_scale > 0.0f))
            RNNT_TRY(cudaMemsetAsync(m.Am, 0, ((int64_t)N * T + V) * sizeof(float), s), RNNT_STATUS_GATHER_FAILED);
        RNNT_TRY(launch_simple_smoothed_forward(s, m), RNNT_STATUS_GATHER_FAILED);
    }
    c.pairs = w.pairs; c.pair_grads = reinterpret_cast<float2 *>(pair_grads);
    return run_typed(s, workspace, workspace_bytes, w, c, rnnt_type, delay_penalty, raw_blank_grads);
}

int rnnt_b200_simple_smoothed_backward(void *stream, void *workspace, size_t workspace_bytes, const float *am,
                                       const float *lm, const int *labels, const int *xn, const int *yn,
                                       const float *saved, const float *pair_grads, const float *grad_out, float *dam,
                                       float *dlm, int N, int T, int U, int V, int blank, float lm_only_scale,
                                       float am_only_scale) {
    if (!simple_args_ok(N, T, U, V, blank) || !smooth_scales_ok(lm_only_scale, am_only_scale) || !saved ||
        !pair_grads || !pairs_aligned(pair_grads) || !dam || !dlm || !pairs_aligned(workspace))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    SimpleArgs a = simple_call(am, lm, labels, xn, yn, const_cast<float *>(saved), N, T, U, V, blank);
    a.pg = reinterpret_cast<const float2 *>(pair_grads);
    a.grad_out = grad_out;
    if (!smoothed(lm_only_scale, am_only_scale)) {
        RNNT_TRY(launch_simple_backward((cudaStream_t)stream, a, dam, dlm, N), RNNT_STATUS_GRADS_BLANK_FAILED);
        return RNNT_STATUS_SUCCESS;
    }
    if (!workspace || workspace_bytes < rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, V))
        return RNNT_STATUS_WORKSPACE_TOO_SMALL;
    SmoothArgs m = smooth_call(a, carve_smooth(workspace, N, T, U, V), const_cast<float *>(saved), N, lm_only_scale,
                               am_only_scale);
    m.pg = a.pg;
    m.grad_out = grad_out;
    RNNT_TRY(launch_simple_smoothed_backward((cudaStream_t)stream, a, m, dam, dlm), RNNT_STATUS_GRADS_BLANK_FAILED);
    return RNNT_STATUS_SUCCESS;
}

int rnnt_b200_prune_ranges(void *stream, const float *pair_grads, const int *xn, const int *yn, int N, int T, int U,
                           int S, int *ranges) {
    return rnnt_b200_prune_ranges_ex(stream, pair_grads, nullptr, xn, yn, N, T, U, S, 0, ranges);
}

int rnnt_b200_prune_ranges_ex(void *stream, const float *pair_grads, const float *raw_blank_grads, const int *xn,
                              const int *yn, int N, int T, int U, int S, int rnnt_type, int *ranges) {
    if (!simple_args_ok(N, T, U, 1, 0) || rnnt_type < 0 || rnnt_type > 2 || S < (rnnt_type == 0 ? 2 : 1) ||
        !pair_grads || !pairs_aligned(pair_grads) || !ranges || (rnnt_type == 2 && !raw_blank_grads))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    RNNT_TRY(launch_prune_ranges((cudaStream_t)stream, reinterpret_cast<const float2 *>(pair_grads), raw_blank_grads, xn,
                                 yn, N, T, U, S, rnnt_type, ranges),
             RNNT_STATUS_GATHER_FAILED);
    return RNNT_STATUS_SUCCESS;
}

size_t rnnt_b200_align_workspace_bytes(int64_t cells, int N, int T, int U) {
    return carve_align(nullptr, cells, N, T, U).bytes;
}

int rnnt_b200_align_dense(void *stream, void *workspace, size_t workspace_bytes, const void *log_probs,
                          const int *labels, const int *xn, const int *yn, float *scores, int *frames, int N, int T,
                          int U, int V, int blank, int elem_bytes) {
    if ((elem_bytes != 4 && elem_bytes != 2) || !dense_args_ok(N, T, U, V, blank) ||
        (reinterpret_cast<uintptr_t>(log_probs) & (uintptr_t)(elem_bytes - 1)))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    AlignCall c = {};
    c.p = {xn, yn, nullptr, nullptr, N, T, U, 0};
    c.T = T; c.U = U; c.cells = (int64_t)N * T * U;
    c.lp = log_probs; c.labels = labels; c.V = V; c.blank = blank; c.io_bf16 = elem_bytes == 2;
    c.scores = scores; c.frames = frames;
    return run_align((cudaStream_t)stream, workspace, workspace_bytes, c);
}

int rnnt_b200_align_compact(void *stream, void *workspace, size_t workspace_bytes, const void *log_probs,
                            const int *labels, const int *xn, const int *yn, float *scores, int *frames, int64_t STU,
                            int N, int V, int blank, int elem_bytes, int max_T, int max_U) {
    if ((elem_bytes != 4 && elem_bytes != 2) || !compact_args_ok(N, STU, V, blank) || max_T <= 0 || max_U <= 0 ||
        (reinterpret_cast<uintptr_t>(log_probs) & (uintptr_t)(elem_bytes - 1)))
        return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0) return RNNT_STATUS_SUCCESS;
    AlignCall c = {};
    c.p = {xn, yn, nullptr, nullptr, N, 0, 0, 1};
    c.T = max_T; c.U = max_U; c.cells = STU;
    c.lp = log_probs; c.labels = labels; c.V = V; c.blank = blank; c.io_bf16 = elem_bytes == 2;
    c.scores = scores; c.frames = frames;
    return run_align((cudaStream_t)stream, workspace, workspace_bytes, c);
}

size_t rnnt_b200_align_logits_workspace_bytes(int64_t cells, int N, int T, int U) {
    return align_logits_bytes(cells, N, T, U);
}

int rnnt_b200_align_logits_dense(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                 const int *labels, const int *xn, const int *yn, float *scores, int *frames, int N,
                                 int T, int U, int V, int blank, int elem_bytes, int rnnt_type, float delay_penalty) {
    return align_logits_dense_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, scores, frames, N, T, U,
                                  V, blank, elem_bytes, rnnt_type, delay_penalty, 0);
}

int rnnt_b200_align_logits_compact(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                   const int *labels, const int *xn, const int *yn, float *scores, int *frames,
                                   int64_t STU, int N, int V, int blank, int elem_bytes, int max_T, int max_U) {
    return align_logits_compact_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, scores, frames, STU, N,
                                    V, blank, elem_bytes, max_T, max_U, 0);
}

int rnnt_b200_align_logits_hat_dense(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                     const int *labels, const int *xn, const int *yn, float *scores, int *frames,
                                     int N, int T, int U, int V, int blank, int elem_bytes, int rnnt_type,
                                     float delay_penalty) {
    return align_logits_dense_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, scores, frames, N, T, U,
                                  V, blank, elem_bytes, rnnt_type, delay_penalty, 1);
}

int rnnt_b200_align_logits_hat_compact(void *stream, void *workspace, size_t workspace_bytes, const void *logits,
                                       const int *labels, const int *xn, const int *yn, float *scores, int *frames,
                                       int64_t STU, int N, int V, int blank, int elem_bytes, int max_T, int max_U) {
    return align_logits_compact_any(stream, workspace, workspace_bytes, logits, labels, xn, yn, scores, frames, STU, N,
                                    V, blank, elem_bytes, max_T, max_U, 1);
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
    if (!compact_args_ok(N, STU, V, blank) || !pairs_aligned(pair_grads)) return RNNT_STATUS_INVALID_ARGUMENT;
    if (N == 0 || STU == 0) return RNNT_STATUS_SUCCESS;
    Problem p = {nullptr, nullptr, nullptr, nullptr, N, 0, 0, 1};
    ExpandSrc src = {};
    src.pg = reinterpret_cast<const float2 *>(pair_grads);
    src.scale = grad_cost;
    src.loc = loc;
    src.cum_lens = cum_lens;
    RNNT_TRY(launch_expand((cudaStream_t)stream, p, src, out, STU, V, blank, false, 0), RNNT_STATUS_GRADS_BLANK_FAILED);
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
    if (!dense_args_ok(N, T, U, V, blank)) return RNNT_STATUS_WARP_FAILED;
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
    if (launch_gather(s, p, log_probs, labels, V, blank, pairs, nullptr, cells, 0) != cudaSuccess)
        status = RNNT_STATUS_WARP_FAILED;
    if (!status && launch_wavefront(s, fast_lse(RNNT_LSE_AUTO), p, pairs, alphas, betas, ll, bad, costs, 0, T, U) !=
                       cudaSuccess)
        status = RNNT_STATUS_WARP_FAILED;
    if (!status) {
        ExpandSrc src = {};
        src.pairs = pairs; src.alphas = alphas; src.betas = betas; src.bad = bad;
        src.labels = labels; src.fastemit_lambda = fastemit_lambda;
        if (launch_expand(s, p, src, grads, cells, V, blank, false, 0) != cudaSuccess)
            status = RNNT_STATUS_GRADS_BLANK_FAILED;
    }
    cudaFreeAsync(tmp, s);
    return status;
}

int run_warp_rnnt_gather(void *stream, unsigned int *counts, float *alphas, float *betas, const float *log_probs,
                         float *grads, float *costs, const int *xn, const int *yn, int N, int T, int U,
                         float fastemit_lambda) {
    (void)counts;
    if (!dense_args_ok(N, T, U, 2, 0)) return RNNT_STATUS_WARP_FAILED;
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
    if (launch_wavefront(s, fast_lse(RNNT_LSE_AUTO), p, pr, alphas, betas, ll, bad, costs, 0, T, U) != cudaSuccess)
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
                             reinterpret_cast<int64_t *>(loc), (int64_t)N * T * U, 0) == cudaSuccess;
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
    ok = ok && launch_wavefront(s, fast_lse(RNNT_LSE_AUTO), p, pr, alphas, betas, ll, nullptr, costs,
                                required_grad ? 0 : 1, (int)T, (int)U) == cudaSuccess;
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
