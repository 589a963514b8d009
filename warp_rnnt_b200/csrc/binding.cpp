// binding.cpp -- the `_C` operator module: PyTorch tensors in, librnnt_b200.so (C ABI) underneath.
//
// Mirrors the reference's operator boundary the reference's pytorch_binding/binding.cpp:
//   rnnt_loss                  (:28-106, pybind :250-254)   same kwargs, checks, messages, returns
//   rnnt_loss_compact          (:109-207, pybind :256-262)
//   rnnt_loss_compact_backward (:209-247, pybind :264-268)
// Differences that are deliberate: a device guard and the *current* stream are used everywhere
// (the reference sets no guard for the dense path, :77, and launches compact kernels on the legacy
// default stream, core.h:41-60); no dense zeros_like / torch::zeros passes (the kernels write every
// element); compact shapes are validated with one small device->host copy instead of four .item()s.
// Extra entry points (rnnt_loss_dense, rnnt_gather_forward/backward) serve the fused python-level
// paths of warp_rnnt_b200/__init__.py.
#include <algorithm>
#include <limits>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include "../../include/rnnt_b200.h"

namespace {

// ---- argument checks ------------------------------------------------------------------------------------------
// Every tensor argument must be on the device of the call's primary tensor (xs, am, grad_cost, grads, pair_grads, f
// or dx), which must be a CUDA device: the kernels run there, under its device guard.  Messages are the callers',
// passed through unformatted, so a call that passes its checks builds no string.

enum class Dt { F32, F32orBF16, I32, I64 };

bool has_dtype(const at::Tensor &t, Dt dt) {
    const at::ScalarType s = t.scalar_type();
    switch (dt) {
    case Dt::F32: return s == at::ScalarType::Float;
    case Dt::F32orBF16: return s == at::ScalarType::Float || s == at::ScalarType::BFloat16;
    case Dt::I32: return s == at::ScalarType::Int;
    case Dt::I64: return s == at::ScalarType::Long;
    }
    return false;
}

// on the device of `on`, a CUDA device (`on` may be `t` itself: then t is on any CUDA device)
bool on_device(const at::Tensor &t, const at::Tensor &on) { return t.device() == on.device() && on.device().is_cuda(); }

// contiguous, of dtype `dt`, on the device of `on`
bool is_arg(const at::Tensor &t, Dt dt, const at::Tensor &on) {
    return t.is_contiguous() && has_dtype(t, dt) && on_device(t, on);
}

constexpr int64_t kAny = std::numeric_limits<int64_t>::min();   // a size that matches any extent

bool has_sizes(const at::Tensor &t, at::IntArrayRef sizes) {
    if (t.dim() != (int64_t)sizes.size()) return false;
    for (size_t d = 0; d < sizes.size(); ++d)
        if (sizes[d] != kAny && t.size(d) != sizes[d]) return false;
    return true;
}

// is_arg, and `numel` elements
void check_arg(const at::Tensor &t, Dt dt, const at::Tensor &on, int64_t numel, const char *msg) {
    TORCH_CHECK(is_arg(t, dt, on) && t.numel() == numel, msg);
}

// is_arg, and of shape `sizes` (kAny: any extent)
void check_arg(const at::Tensor &t, Dt dt, const at::Tensor &on, at::IntArrayRef sizes, const char *msg) {
    TORCH_CHECK(is_arg(t, dt, on) && has_sizes(t, sizes), msg);
}

// an optional tensor argument: null when absent, else checked as check_arg does and its data
template <typename T>
const T *optional_arg(const c10::optional<at::Tensor> &t, Dt dt, const at::Tensor &on, int64_t numel,
                      const char *msg) {
    if (!t.has_value() || !t->defined()) return nullptr;
    check_arg(*t, dt, on, numel, msg);
    return t->data_ptr<T>();
}

void check_blank(int blank, int64_t V) { TORCH_CHECK(blank >= 0 && blank < V, "blank must be in [0, V)"); }
// the HAT normalisation (hat = true) needs a label column besides the blank
void check_hat(bool hat, int64_t V) { TORCH_CHECK(!hat || V >= 2, "hat needs V >= 2"); }
int elem_bytes(const at::Tensor &xs) { return xs.scalar_type() == at::ScalarType::BFloat16 ? 2 : 4; }

void check4(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
            bool allow_bf16 = false) {
    // order as in the reference (binding.cpp:31-46): contiguity, then dtypes, then device; then the device of xs
    TORCH_CHECK(xs.is_contiguous(), "xs must be contiguous");
    TORCH_CHECK(ys.is_contiguous(), "ys must be contiguous");
    TORCH_CHECK(xn.is_contiguous(), "xn must be contiguous");
    TORCH_CHECK(yn.is_contiguous(), "yn must be contiguous");
    TORCH_CHECK(xs.scalar_type() == at::ScalarType::Float || (allow_bf16 && xs.scalar_type() == at::ScalarType::BFloat16),
                "xs must be a Float tensor");
    TORCH_CHECK(ys.scalar_type() == at::ScalarType::Int, "ys must be a Int tensor");
    TORCH_CHECK(xn.scalar_type() == at::ScalarType::Int, "xn must be a Int tensor");
    TORCH_CHECK(yn.scalar_type() == at::ScalarType::Int, "yn must be a Int tensor");
    TORCH_CHECK(xs.device().is_cuda(), "xs must be located in the CUDA");
    TORCH_CHECK(ys.device().is_cuda(), "ys must be located in the CUDA");
    TORCH_CHECK(xn.device().is_cuda(), "xn must be located in the CUDA");
    TORCH_CHECK(yn.device().is_cuda(), "yn must be located in the CUDA");
    TORCH_CHECK(ys.device() == xs.device(), "ys must be on the device of xs");
    TORCH_CHECK(xn.device() == xs.device(), "xn must be on the device of xs");
    TORCH_CHECK(yn.device() == xs.device(), "yn must be on the device of xs");
}

// xs (N, ...) with 4 dimensions, xn and yn (N,)
void check_batch4(const at::Tensor &xs, const at::Tensor &xn, const at::Tensor &yn) {
    TORCH_CHECK(xs.dim() == 4, "xs must have 4 dimensions");
    TORCH_CHECK(xn.numel() == xs.size(0), "xn shape must be equal (N,)");
    TORCH_CHECK(yn.numel() == xs.size(0), "yn shape must be equal (N,)");
}

// The front of a dense (N,T,U,V) call: check4, the shapes, then the device guard of xs, held by the caller.
struct DenseFront {
    int64_t N, T, U, V;
    bool bf16;
    c10::cuda::CUDAGuard guard;
};

DenseFront dense_front(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                       bool allow_bf16) {
    check4(xs, ys, xn, yn, allow_bf16);
    check_batch4(xs, xn, yn);
    TORCH_CHECK(ys.dim() == 2 && xs.size(2) == ys.size(1) + 1, "ys shape (N, U-1) mismatched with xs (N, T, U, V)");
    return {xs.size(0), xs.size(1), xs.size(2), xs.size(3), xs.scalar_type() == at::ScalarType::BFloat16,
            c10::cuda::CUDAGuard(xs.device())};
}

// The front of a compact (STU,V) call: check4, the shapes and blank, then the device guard of xs, held by the caller.
struct CompactFront {
    int64_t N, STU, V;
    bool bf16;
    c10::cuda::CUDAGuard guard;
};

CompactFront compact_front(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                           int blank, bool allow_bf16) {
    check4(xs, ys, xn, yn, allow_bf16);
    TORCH_CHECK(xs.dim() == 2, "xs must have 2 dimensions");
    TORCH_CHECK(xn.dim() == 1 && yn.dim() == 1 && xn.size(0) == yn.size(0), "xn and yn shape must be equal (N,)");
    check_blank(blank, xs.size(1));
    return {xn.size(0), xs.size(0), xs.size(1), xs.scalar_type() == at::ScalarType::BFloat16,
            c10::cuda::CUDAGuard(xs.device())};
}

// ---- outputs, workspaces, launches ----------------------------------------------------------------------------

// an output the caller asked for, or the empty placeholder returned in its place
at::Tensor output(bool want, at::IntArrayRef sizes, const at::TensorOptions &options) {
    return want ? at::empty(sizes, options) : at::empty({0}, options);
}

at::Tensor workspace(const at::Tensor &like, size_t bytes) {
    return at::empty({(int64_t)bytes}, like.options().dtype(at::kByte));
}

void check_status(int status) {
    TORCH_CHECK(status == RNNT_STATUS_SUCCESS, "rnnt_loss status ", status, " (", rnnt_b200_status_string(status), ")");
}

void *current_stream(const at::Tensor &t) {
    return (void *)c10::cuda::getCurrentCUDAStream(t.device().index()).stream();
}

// Tickets for the in-kernel loss reduction (rnnt_b200_loss_dense_reduced): a small ring of self-resetting device
// counters per device, zeroed once; consecutive calls take consecutive slots so that calls running concurrently
// on different streams (or captured into different CUDA graphs) never share one.
unsigned int *next_sync_counter(const at::Tensor &like) {
    constexpr int kSlots = 256, kMaxDev = 64;
    static std::mutex mu;
    static at::Tensor ring[kMaxDev];
    static unsigned next[kMaxDev] = {};
    const int dev = like.device().index();
    if (dev < 0 || dev >= kMaxDev) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    if (!ring[dev].defined()) ring[dev] = at::zeros({kSlots}, like.options().dtype(at::kInt));
    return reinterpret_cast<unsigned int *>(ring[dev].data_ptr<int>()) + (next[dev]++ % kSlots);
}

// Upper bounds (max_T, max_U) of the lattices of a compact call: the caller's hints when both are positive (no host
// sync, CUDA-graph capturable), else one 16-byte device->host copy of the device totals (the reference needs four
// .item() syncs), which also checks ys and xs against xn and yn.  scratch: (2N) int64 for the prefix sums, or null.
std::pair<int, int> compact_bounds(void *stream, const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                   const at::Tensor &yn, int hint_T, int hint_U, int64_t *scratch) {
    if (hint_T > 0 && hint_U > 0) return {hint_T, hint_U};
    const int64_t N = xn.size(0);
    at::Tensor own;
    if (!scratch) {
        own = at::empty({2 * N}, xs.options().dtype(at::kLong));
        scratch = own.data_ptr<int64_t>();
    }
    at::Tensor totals = at::empty({4}, xs.options().dtype(at::kInt));
    check_status(rnnt_b200_compact_totals(stream, xn.data_ptr<int>(), yn.data_ptr<int>(), (int)N, scratch,
                                          totals.data_ptr<int>()));
    at::Tensor h = totals.cpu();
    const int *t = h.data_ptr<int>();
    TORCH_CHECK(ys.numel() == t[1], "ys shape must be equal to (sum(yn), )");
    TORCH_CHECK(xs.size(0) == t[0], "xs shape mismatch with (\\sum{xn*(yn+1)}, )");
    return {t[2], t[3]};
}

// dense forward (+ gradients), optional per-sample scale, explicit LSE mode; loss_sum: (1) tensor or undefined
std::tuple<at::Tensor, at::Tensor> loss_dense_impl(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                                   const at::Tensor &yn, int blank, float fastemit_lambda,
                                                   const c10::optional<at::Tensor> &scale, bool want_grads,
                                                   int lse_mode, at::Tensor loss_sum = at::Tensor(),
                                                   bool allow_bf16 = false) {
    const auto [N, T, U, V, bf16, guard] = dense_front(xs, ys, xn, yn, allow_bf16);
    at::Tensor costs = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor grads = output(want_grads, xs.sizes(), xs.options());
    if (N == 0) return std::make_tuple(costs, grads);
    TORCH_CHECK(!bf16 || (want_grads && blank != -1), "bfloat16 xs: dense (N,T,U,V) layout with gradients only");
    const float *sc = optional_arg<float>(scale, Dt::F32, xs, N,
                                          "grad_scale must be a contiguous Float tensor of shape (N,) on the device of xs");
    if (blank == -1) {
        TORCH_CHECK(V == 2, "xs must have values only for blank and label");    // gathered (N,T,U,2) form, binding.cpp:81-90
    } else {
        TORCH_CHECK(blank >= 0 && blank < V, "blank must be in [0, V) (or -1 for the gathered layout)");
    }
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(N * T * U, (int)N));
    float *ls = loss_sum.defined() ? loss_sum.data_ptr<float>() : nullptr;
    unsigned int *counter = ls ? next_sync_counter(xs) : nullptr;
    if (blank == -1) {
        check_status(rnnt_b200_loss_pairs(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr<float>(),
                                          xn.data_ptr<int>(), yn.data_ptr<int>(), costs.data_ptr<float>(),
                                          want_grads ? grads.data_ptr<float>() : nullptr, (int)N, (int)T, (int)U,
                                          fastemit_lambda, lse_mode));
        if (want_grads && sc) grads.mul_(scale->view({-1, 1, 1, 1}));
    } else if (bf16) {
        check_status(rnnt_b200_loss_dense_bf16(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(),
                                               ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(),
                                               costs.data_ptr<float>(), grads.data_ptr(), sc, ls, counter, (int)N,
                                               (int)T, (int)U, (int)V, blank, fastemit_lambda, lse_mode));
    } else {
        check_status(rnnt_b200_loss_dense_reduced(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(),
                                                  xs.data_ptr<float>(), ys.data_ptr<int>(), xn.data_ptr<int>(),
                                                  yn.data_ptr<int>(), costs.data_ptr<float>(),
                                                  want_grads ? grads.data_ptr<float>() : nullptr, sc, ls, counter,
                                                  (int)N, (int)T, (int)U, (int)V, blank, fastemit_lambda, lse_mode));
    }
    return std::make_tuple(costs, grads);
}

// ---- reference-compatible entry points --------------------------------------------------

std::tuple<at::Tensor, at::Tensor> rnnt_loss(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                             const at::Tensor &yn, const int blank, const float fastemit_lambda) {
    return loss_dense_impl(xs, ys, xn, yn, blank, fastemit_lambda, c10::nullopt, true, RNNT_LSE_AUTO);
}

std::tuple<at::Tensor, at::Tensor, at::Tensor> rnnt_loss_compact(const at::Tensor &xs, const at::Tensor &ys,
                                                                 const at::Tensor &xn, const at::Tensor &yn,
                                                                 const int blank, const float fastemit_lambda,
                                                                 const bool required_grad, int hint_T, int hint_U) {
    const auto [N, STU, V, bf16, guard] = compact_front(xs, ys, xn, yn, blank, false);
    void *stream = current_stream(xs);
    at::Tensor costs = at::empty({N}, xs.options());
    at::Tensor loc = at::empty({STU}, xs.options().dtype(at::kLong));
    // like the reference (binding.cpp:196-201): without required_grad the returned "grads" is a
    // placeholder the caller must not use
    at::Tensor grads = output(required_grad, {STU, 2}, xs.options());
    if (N == 0) return std::make_tuple(costs, grads, loc);
    const auto [max_T, max_U] = compact_bounds(stream, xs, ys, xn, yn, hint_T, hint_U, nullptr);
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(STU, (int)N));
    check_status(rnnt_b200_compact_forward(stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr<float>(),
                                           ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(),
                                           costs.data_ptr<float>(), required_grad ? grads.data_ptr<float>() : nullptr,
                                           loc.data_ptr<int64_t>(), nullptr, STU, (int)N, (int)V, blank,
                                           fastemit_lambda, RNNT_LSE_AUTO, max_T, max_U));
    return std::make_tuple(costs, grads, loc);
}

at::Tensor rnnt_loss_compact_backward(const at::Tensor &grad_cost, const at::Tensor &grad_xs,
                                      const at::Tensor &cum_lens, const at::Tensor &loc, int64_t V, int blank) {
    // order as in the reference (binding.cpp:212-221): contiguity, then dtypes, then device; then the device of
    // grad_cost
    TORCH_CHECK(grad_cost.is_contiguous(), "grad_cost must be contiguous");
    TORCH_CHECK(grad_xs.is_contiguous(), "grad_xs must be contiguous");
    TORCH_CHECK(loc.is_contiguous(), "loc must be contiguous");
    TORCH_CHECK(grad_cost.scalar_type() == at::ScalarType::Float, "grad_cost must be a Float tensor");
    TORCH_CHECK(grad_xs.scalar_type() == at::ScalarType::Float, "grad_xs must be a Float tensor");
    TORCH_CHECK(loc.scalar_type() == at::ScalarType::Long, "loc must be a Long tensor");
    TORCH_CHECK(grad_cost.device().is_cuda(), "grad_cost must be located in the CUDA");
    TORCH_CHECK(grad_xs.device().is_cuda(), "grad_xs must be located in the CUDA");
    TORCH_CHECK(cum_lens.device().is_cuda(), "cum_lens must be located in the CUDA");
    TORCH_CHECK(loc.device().is_cuda(), "loc must be located in the CUDA");
    TORCH_CHECK(grad_xs.device() == grad_cost.device(), "grad_xs must be on the device of grad_cost");
    TORCH_CHECK(cum_lens.device() == grad_cost.device(), "cum_lens must be on the device of grad_cost");
    TORCH_CHECK(loc.device() == grad_cost.device(), "loc must be on the device of grad_cost");
    TORCH_CHECK(grad_cost.dim() == 1, "grad_cost must have 1 dimensions");
    TORCH_CHECK(grad_xs.dim() == 2, "grad must have 2 dimensions");
    TORCH_CHECK(grad_xs.size(0) == loc.size(0), "grad and loc must be equal in dim=0");
    TORCH_CHECK(cum_lens.is_contiguous() && cum_lens.scalar_type() == at::ScalarType::Int &&
                    cum_lens.numel() == grad_cost.size(0),
                "cum_lens must be a contiguous Int tensor of shape (N,)");
    TORCH_CHECK(grad_xs.size(1) == 2, "grad must have shape (STU, 2)");
    check_blank(blank, V);
    const c10::cuda::CUDAGuard guard(grad_cost.device());
    const int64_t N = grad_cost.size(0), STU = grad_xs.size(0);
    at::Tensor out = at::empty({STU, V}, grad_cost.options());
    check_status(rnnt_b200_compact_backward(current_stream(grad_cost), grad_cost.data_ptr<float>(),
                                            grad_xs.data_ptr<float>(), loc.data_ptr<int64_t>(),
                                            cum_lens.data_ptr<int>(), out.data_ptr<float>(), STU, (int)N, (int)V,
                                            blank));
    return out;
}

// ---- native extras used by warp_rnnt_b200/__init__.py ------------------------------------

std::tuple<at::Tensor, at::Tensor> rnnt_loss_dense(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                                   const at::Tensor &yn, int blank, float fastemit_lambda,
                                                   const c10::optional<at::Tensor> &grad_scale, bool want_grads,
                                                   int lse_mode) {
    return loss_dense_impl(xs, ys, xn, yn, blank, fastemit_lambda, grad_scale, want_grads, lse_mode);
}

// loss + dense gradients + reduced loss in one call: (costs (N), grads like xs or empty, loss (1) = sum costs*scale)
std::tuple<at::Tensor, at::Tensor, at::Tensor> rnnt_loss_fused(const at::Tensor &xs, const at::Tensor &ys,
                                                               const at::Tensor &xn, const at::Tensor &yn, int blank,
                                                               float fastemit_lambda,
                                                               const c10::optional<at::Tensor> &grad_scale,
                                                               bool want_grads, int lse_mode) {
    TORCH_CHECK(blank >= 0, "rnnt_loss_fused takes the dense (N,T,U,V) layout");
    TORCH_CHECK(xs.device().is_cuda(), "xs must be located in the CUDA");
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor loss = at::empty({1}, xs.options().dtype(at::kFloat));
    if (xs.dim() == 4 && xs.size(0) == 0) loss.zero_();
    auto r = loss_dense_impl(xs, ys, xn, yn, blank, fastemit_lambda, grad_scale, want_grads, lse_mode, loss, true);
    return std::make_tuple(std::get<0>(r), std::get<1>(r), loss);
}

// in place: grads[n] *= grad_out[n] / applied[n] where they differ (grad_out with one element: one scalar for all)
void rnnt_rescale_(at::Tensor grads, const at::Tensor &grad_out, const c10::optional<at::Tensor> &applied) {
    TORCH_CHECK(is_arg(grads, Dt::F32orBF16, grads) && grads.dim() >= 1,
                "grads must be a contiguous CUDA Float (or BFloat16) tensor");
    const int64_t N = grads.size(0);
    TORCH_CHECK(is_arg(grad_out, Dt::F32, grads) && (grad_out.numel() == N || grad_out.numel() == 1),
                "grad_out must be a contiguous Float tensor with N elements (or one) on the device of grads");
    const float *ap = optional_arg<float>(applied, Dt::F32, grads, N,
                                          "applied must be a contiguous Float tensor of shape (N,) on the device of grads");
    if (N == 0) return;
    const c10::cuda::CUDAGuard guard(grads.device());
    check_status(rnnt_b200_rescale(current_stream(grads), grads.data_ptr(), grad_out.data_ptr<float>(),
                                   (grad_out.numel() == 1 && N != 1) ? 0 : 1, ap, (int)N, grads.numel() / N,
                                   grads.scalar_type() == at::ScalarType::BFloat16 ? 2 : 4));
}

std::tuple<at::Tensor, at::Tensor> rnnt_gather_forward(const at::Tensor &xs, const at::Tensor &ys,
                                                       const at::Tensor &xn, const at::Tensor &yn, int blank,
                                                       float fastemit_lambda, bool want_grads, int lse_mode) {
    const auto [N, T, U, V, bf16, guard] = dense_front(xs, ys, xn, yn, false);
    check_blank(blank, V);
    at::Tensor costs = at::empty({N}, xs.options());
    at::Tensor pg = output(want_grads, {N, T, U, 2}, xs.options());
    if (N == 0) return std::make_tuple(costs, pg);
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(N * T * U, (int)N));
    check_status(rnnt_b200_gather_forward(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(),
                                          xs.data_ptr<float>(), ys.data_ptr<int>(), xn.data_ptr<int>(),
                                          yn.data_ptr<int>(), costs.data_ptr<float>(),
                                          want_grads ? pg.data_ptr<float>() : nullptr, (int)N, (int)T, (int)U, (int)V,
                                          blank, fastemit_lambda, lse_mode));
    return std::make_tuple(costs, pg);
}

// loss from un-normalised logits: (costs (N), lse (N,T,U), pair_grads (N,T,U,2) or empty), all float32 also for
// bfloat16 logits
std::tuple<at::Tensor, at::Tensor, at::Tensor> rnnt_logits_forward(const at::Tensor &xs, const at::Tensor &ys,
                                                                   const at::Tensor &xn, const at::Tensor &yn,
                                                                   int blank, float fastemit_lambda, bool want_grads,
                                                                   int lse_mode, int rnnt_type, double delay_penalty,
                                                                   bool hat) {
    const auto [N, T, U, V, bf16, guard] = dense_front(xs, ys, xn, yn, true);
    check_blank(blank, V);
    check_hat(hat, V);
    const auto f32 = xs.options().dtype(at::kFloat);
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor lse = at::empty({N, T, U}, f32);
    at::Tensor pg = output(want_grads, {N, T, U, 2}, f32);
    if (N == 0) return std::make_tuple(costs, lse, pg);
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(N * T * U, (int)N));
    float *pgp = want_grads ? pg.data_ptr<float>() : nullptr;
    if (hat)
        check_status(rnnt_b200_logits_hat_forward(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(),
                                                  ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(),
                                                  costs.data_ptr<float>(), lse.data_ptr<float>(), pgp, (int)N, (int)T,
                                                  (int)U, (int)V, blank, fastemit_lambda, lse_mode, bf16 ? 2 : 4,
                                                  rnnt_type, (float)delay_penalty));
    else if (bf16)
        check_status(rnnt_b200_logits_forward_bf16_ex(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(),
                                                      xs.data_ptr(), ys.data_ptr<int>(), xn.data_ptr<int>(),
                                                      yn.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(),
                                                      pgp, (int)N, (int)T, (int)U, (int)V, blank, fastemit_lambda,
                                                      lse_mode, rnnt_type, (float)delay_penalty));
    else
        check_status(rnnt_b200_logits_forward_ex(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(),
                                                 xs.data_ptr<float>(), ys.data_ptr<int>(), xn.data_ptr<int>(),
                                                 yn.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(), pgp,
                                                 (int)N, (int)T, (int)U, (int)V, blank, fastemit_lambda, lse_mode,
                                                 rnnt_type, (float)delay_penalty));
    return std::make_tuple(costs, lse, pg);
}

// d loss / d logits, of the dtype of xs (float32 or bfloat16)
at::Tensor rnnt_logits_backward(const at::Tensor &xs, const at::Tensor &lse, const at::Tensor &pair_grads,
                                const at::Tensor &ys, const at::Tensor &grad_out, int blank, bool hat) {
    check_arg(xs, Dt::F32orBF16, xs, {kAny, kAny, kAny, kAny},
              "xs must be a contiguous CUDA Float tensor of shape (N, T, U, V)");
    const int64_t N = xs.size(0), T = xs.size(1), U = xs.size(2), V = xs.size(3);
    check_arg(lse, Dt::F32, xs, N * T * U, "lse must be a contiguous Float tensor of shape (N, T, U) on the device of xs");
    check_arg(pair_grads, Dt::F32, xs, N * T * U * 2,
              "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of xs");
    check_arg(ys, Dt::I32, xs, {N, U - 1}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs");
    check_arg(grad_out, Dt::F32, xs, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    check_blank(blank, V);
    check_hat(hat, V);
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor out = at::empty_like(xs);
    if (hat)
        check_status(rnnt_b200_logits_hat_backward(current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(),
                                                   pair_grads.data_ptr<float>(), ys.data_ptr<int>(),
                                                   grad_out.data_ptr<float>(), out.data_ptr(), (int)N, (int)T, (int)U,
                                                   (int)V, blank, elem_bytes(xs)));
    else if (xs.scalar_type() == at::ScalarType::BFloat16)
        check_status(rnnt_b200_logits_backward_bf16(current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(),
                                                    pair_grads.data_ptr<float>(), ys.data_ptr<int>(),
                                                    grad_out.data_ptr<float>(), out.data_ptr(), (int)N, (int)T, (int)U,
                                                    (int)V, blank));
    else
        check_status(rnnt_b200_logits_backward(current_stream(xs), xs.data_ptr<float>(), lse.data_ptr<float>(),
                                               pair_grads.data_ptr<float>(), ys.data_ptr<int>(), grad_out.data_ptr<float>(),
                                               out.data_ptr<float>(), (int)N, (int)T, (int)U, (int)V, blank));
    return out;
}

// loss from compact (STU,V) logits in joint_pack's row order, float32 or bfloat16: (costs (N), lse (STU),
// pair_grads (STU,2) or empty, prefix (2N) int64 = {mem_pref, lab_pref} for the backward).  Shapes are validated as in
// rnnt_loss_compact: one 16-byte device->host copy, or none with hints (max_T, max_U > 0).
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor>
rnnt_logits_compact_forward(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                            int blank, float fastemit_lambda, bool want_grads, int lse_mode, int max_T, int max_U,
                            bool hat) {
    const auto [N, STU, V, bf16, guard] = compact_front(xs, ys, xn, yn, blank, true);
    check_hat(hat, V);
    void *stream = current_stream(xs);
    const auto f32 = xs.options().dtype(at::kFloat);
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor lse = at::empty({STU}, f32);
    at::Tensor pg = output(want_grads, {STU, 2}, f32);
    at::Tensor prefix = at::empty({2 * N}, xs.options().dtype(at::kLong));
    if (N == 0) return std::make_tuple(costs, lse, pg, prefix);
    std::tie(max_T, max_U) = compact_bounds(stream, xs, ys, xn, yn, max_T, max_U, prefix.data_ptr<int64_t>());
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(STU, (int)N));
    float *pgp = want_grads ? pg.data_ptr<float>() : nullptr;
    if (hat)
        check_status(rnnt_b200_logits_compact_hat_forward(
            stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(), xn.data_ptr<int>(),
            yn.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(), pgp, prefix.data_ptr<int64_t>(), nullptr,
            STU, (int)N, (int)V, blank, fastemit_lambda, lse_mode, max_T, max_U, bf16 ? 2 : 4));
    else if (bf16)
        check_status(rnnt_b200_logits_compact_forward_bf16(
            stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(), xn.data_ptr<int>(),
            yn.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(), pgp, prefix.data_ptr<int64_t>(), nullptr,
            STU, (int)N, (int)V, blank, fastemit_lambda, lse_mode, max_T, max_U));
    else
        check_status(rnnt_b200_logits_compact_forward(
            stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr<float>(), ys.data_ptr<int>(), xn.data_ptr<int>(),
            yn.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(), pgp, prefix.data_ptr<int64_t>(), nullptr,
            STU, (int)N, (int)V, blank, fastemit_lambda, lse_mode, max_T, max_U));
    return std::make_tuple(costs, lse, pg, prefix);
}

// d loss / d compact logits, of the dtype of xs
at::Tensor rnnt_logits_compact_backward(const at::Tensor &xs, const at::Tensor &lse, const at::Tensor &pair_grads,
                                        const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                                        const at::Tensor &prefix, const at::Tensor &grad_out, int blank, bool hat) {
    check_arg(xs, Dt::F32orBF16, xs, {kAny, kAny}, "xs must be a contiguous CUDA Float tensor of shape (STU, V)");
    const int64_t STU = xs.size(0), V = xs.size(1), N = xn.numel();
    check_arg(lse, Dt::F32, xs, STU, "lse must be a contiguous Float tensor of shape (STU,) on the device of xs");
    check_arg(pair_grads, Dt::F32, xs, STU * 2,
              "pair_grads must be a contiguous Float tensor of shape (STU, 2) on the device of xs");
    TORCH_CHECK(is_arg(ys, Dt::I32, xs), "ys must be a contiguous Int tensor on the device of xs");
    const char *lengths = "xn and yn must be contiguous Int tensors of shape (N,) on the device of xs";
    check_arg(xn, Dt::I32, xs, N, lengths);
    check_arg(yn, Dt::I32, xs, N, lengths);
    check_arg(prefix, Dt::I64, xs, 2 * N, "prefix must be a contiguous Long tensor of shape (2N,) on the device of xs");
    check_arg(grad_out, Dt::F32, xs, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    check_blank(blank, V);
    check_hat(hat, V);
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor out = at::empty_like(xs);
    if (N == 0 || STU == 0) return out;                 // empty tensors: nothing to write (and no data pointers)
    if (hat)
        check_status(rnnt_b200_logits_compact_hat_backward(
            current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(), pair_grads.data_ptr<float>(), ys.data_ptr<int>(),
            xn.data_ptr<int>(), yn.data_ptr<int>(), prefix.data_ptr<int64_t>(), grad_out.data_ptr<float>(),
            out.data_ptr(), STU, (int)N, (int)V, blank, elem_bytes(xs)));
    else if (xs.scalar_type() == at::ScalarType::BFloat16)
        check_status(rnnt_b200_logits_compact_backward_bf16(
            current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(), pair_grads.data_ptr<float>(), ys.data_ptr<int>(),
            xn.data_ptr<int>(), yn.data_ptr<int>(), prefix.data_ptr<int64_t>(), grad_out.data_ptr<float>(),
            out.data_ptr(), STU, (int)N, (int)V, blank));
    else
        check_status(rnnt_b200_logits_compact_backward(
            current_stream(xs), xs.data_ptr<float>(), lse.data_ptr<float>(), pair_grads.data_ptr<float>(),
            ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(), prefix.data_ptr<int64_t>(),
            grad_out.data_ptr<float>(), out.data_ptr<float>(), STU, (int)N, (int)V, blank));
    return out;
}

// pruned loss from (N,T,S,V) window logits, float32 or bfloat16, ranges (N,T): (costs (N), lse (N,T,S), pair_grads
// (N,T,U,2) of the full lattice or empty), all float32; U = ys.size(1) + 1.  No host sync.
std::tuple<at::Tensor, at::Tensor, at::Tensor> rnnt_logits_pruned_forward(const at::Tensor &xs, const at::Tensor &ys,
                                                                          const at::Tensor &xn, const at::Tensor &yn,
                                                                          const at::Tensor &ranges, int blank,
                                                                          float fastemit_lambda, bool want_grads,
                                                                          int lse_mode, int rnnt_type,
                                                                          double delay_penalty, bool hat) {
    check4(xs, ys, xn, yn, true);
    check_batch4(xs, xn, yn);
    TORCH_CHECK(ys.dim() == 2 && ys.size(0) == xs.size(0), "ys shape must be (N, U-1)");
    const int64_t N = xs.size(0), T = xs.size(1), S = xs.size(2), V = xs.size(3), U = ys.size(1) + 1;
    check_arg(ranges, Dt::I32, xs, {N, T}, "ranges must be a contiguous Int tensor of shape (N, T) on the device of xs");
    check_blank(blank, V);
    check_hat(hat, V);
    const c10::cuda::CUDAGuard guard(xs.device());
    const auto f32 = xs.options().dtype(at::kFloat);
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor lse = at::empty({N, T, S}, f32);
    at::Tensor pg = output(want_grads, {N, T, U, 2}, f32);
    if (N == 0) return std::make_tuple(costs, lse, pg);
    at::Tensor ws = workspace(xs, rnnt_b200_workspace_bytes(N * T * U, (int)N));
    const auto forward = hat ? rnnt_b200_logits_pruned_hat_forward : rnnt_b200_logits_pruned_forward_ex;
    check_status(forward(
        current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(), xn.data_ptr<int>(),
        yn.data_ptr<int>(), ranges.data_ptr<int>(), costs.data_ptr<float>(), lse.data_ptr<float>(),
        want_grads ? pg.data_ptr<float>() : nullptr, (int)N, (int)T, (int)S, (int)U, (int)V, blank, fastemit_lambda,
        lse_mode, xs.scalar_type() == at::ScalarType::BFloat16 ? 2 : 4, rnnt_type, (float)delay_penalty));
    return std::make_tuple(costs, lse, pg);
}

// d loss / d pruned logits (N,T,S,V), of the dtype of xs
at::Tensor rnnt_logits_pruned_backward(const at::Tensor &xs, const at::Tensor &lse, const at::Tensor &pair_grads,
                                       const at::Tensor &ys, const at::Tensor &ranges, const at::Tensor &grad_out,
                                       int blank, bool hat) {
    check_arg(xs, Dt::F32orBF16, xs, {kAny, kAny, kAny, kAny},
              "xs must be a contiguous CUDA Float tensor of shape (N, T, S, V)");
    const int64_t N = xs.size(0), T = xs.size(1), S = xs.size(2), V = xs.size(3);
    check_arg(ys, Dt::I32, xs, {N, kAny}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs");
    const int64_t U = ys.size(1) + 1;
    check_arg(lse, Dt::F32, xs, N * T * S, "lse must be a contiguous Float tensor of shape (N, T, S) on the device of xs");
    check_arg(pair_grads, Dt::F32, xs, N * T * U * 2,
              "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of xs");
    check_arg(ranges, Dt::I32, xs, {N, T}, "ranges must be a contiguous Int tensor of shape (N, T) on the device of xs");
    check_arg(grad_out, Dt::F32, xs, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    check_blank(blank, V);
    check_hat(hat, V);
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor out = at::empty_like(xs);
    if (N == 0) return out;
    const auto backward = hat ? rnnt_b200_logits_pruned_hat_backward : rnnt_b200_logits_pruned_backward;
    check_status(backward(current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(), pair_grads.data_ptr<float>(),
                          ys.data_ptr<int>(), ranges.data_ptr<int>(), grad_out.data_ptr<float>(), out.data_ptr(),
                          (int)N, (int)T, (int)S, (int)U, (int)V, blank,
                          xs.scalar_type() == at::ScalarType::BFloat16 ? 2 : 4));
    return out;
}

// ---- TDT and multi-blank --------------------------------------------------------------------------------------
// The Token-and-Duration Transducer (TDT) and the multi-blank transducer share their kernels and the signatures of
// their C ABI calls; a Lattice holds what differs.  D = durations.size().  A TDT row is V token logits then D duration
// logits, blank in [0, V), and its lse holds (lse_tok, lse_dur) per cell; a multi-blank row is V logits with the D big
// blanks below the standard blank, blank in [D, V), and its lse one float per cell.
struct Lattice {
    bool multiblank;
    const char *row_cell, *row_row;           // the row must hold more than D logits: dense, compact
    const char *blank_range;
    const char *xs4, *lse4, *grads4;          // the dense backward's tensors
    const char *xs2, *lse2, *grads2;          // the compact backward's tensors
    decltype(&rnnt_b200_tdt_workspace_bytes) workspace_bytes;
    decltype(&rnnt_b200_tdt_forward) forward;
    decltype(&rnnt_b200_tdt_backward) backward;
    decltype(&rnnt_b200_tdt_compact_workspace_bytes) compact_workspace_bytes;
    decltype(&rnnt_b200_tdt_compact_forward) compact_forward;
    decltype(&rnnt_b200_tdt_compact_backward) compact_backward;
    decltype(&rnnt_b200_tdt_align_workspace_bytes) align_workspace_bytes;
    decltype(&rnnt_b200_tdt_align_dense) align_dense;
    decltype(&rnnt_b200_tdt_align_compact) align_compact;
};

const Lattice kTdt = {
    false, "xs must have more than len(durations) logits per cell (V + D)",
    "xs must have more than len(durations) logits per row (V + D)", "blank must be in [0, V)",
    "xs must be a contiguous CUDA Float tensor of shape (N, T, U, V+D)",
    "lse must be a contiguous Float tensor of shape (N, T, U, 2) on the device of xs",
    "grads must be a contiguous Float tensor of shape (N, T, U, 2+D) on the device of xs",
    "xs must be a contiguous CUDA Float tensor of shape (STU, V+D)",
    "lse must be a contiguous Float tensor of shape (STU, 2) on the device of xs",
    "grads must be a contiguous Float tensor of shape (STU, 2+D) on the device of xs",
    rnnt_b200_tdt_workspace_bytes, rnnt_b200_tdt_forward, rnnt_b200_tdt_backward,
    rnnt_b200_tdt_compact_workspace_bytes, rnnt_b200_tdt_compact_forward, rnnt_b200_tdt_compact_backward,
    rnnt_b200_tdt_align_workspace_bytes, rnnt_b200_tdt_align_dense, rnnt_b200_tdt_align_compact};

const Lattice kMultiblank = {
    true, "xs must have more than len(big_blank_durations) logits per cell",
    "xs must have more than len(big_blank_durations) logits per cell", "blank must be in [len(big_blank_durations), V)",
    "xs must be a contiguous CUDA Float tensor of shape (N, T, U, V)",
    "lse must be a contiguous Float tensor of shape (N, T, U) on the device of xs",
    "grads must be a contiguous Float tensor of shape (N, T, U, 2+B) on the device of xs",
    "xs must be a contiguous CUDA Float tensor of shape (STU, V)",
    "lse must be a contiguous Float tensor of shape (STU,) on the device of xs",
    "grads must be a contiguous Float tensor of shape (STU, 2+B) on the device of xs",
    rnnt_b200_multiblank_workspace_bytes, rnnt_b200_multiblank_forward, rnnt_b200_multiblank_backward,
    rnnt_b200_multiblank_compact_workspace_bytes, rnnt_b200_multiblank_compact_forward,
    rnnt_b200_multiblank_compact_backward, rnnt_b200_multiblank_align_workspace_bytes,
    rnnt_b200_multiblank_align_dense, rnnt_b200_multiblank_align_compact};

// V of a row of W logits, after the row (message `row`) and the blank are checked
int64_t lattice_tokens(const Lattice &F, int64_t W, int64_t D, int blank, const char *row) {
    TORCH_CHECK(D >= 1 && W > D, row);
    const int64_t V = F.multiblank ? W : W - D;
    TORCH_CHECK(blank >= (F.multiblank ? D : 0) && blank < V, F.blank_range);
    return V;
}

// the shape of lse on the given cells
std::vector<int64_t> lse_sizes(const Lattice &F, std::vector<int64_t> cells) {
    if (!F.multiblank) cells.push_back(2);
    return cells;
}

// An (n,) int32 output of the TDT alignment: a view of at least one element, so that the C ABI, which refuses NULL
// outputs, gets a pointer also when there are no label slots (U = 1, or no labels in the batch)
at::Tensor label_slots(int64_t n, const at::Tensor &like) {
    return at::empty({std::max<int64_t>(n, 1)}, like.options().dtype(at::kInt)).narrow(0, 0, n);
}

// the alignment's third output: TDT's label durations, shaped like frames, or multi-blank's blank counts (N, 1 + D)
at::Tensor align_third(const Lattice &F, const at::Tensor &frames, int64_t N, int64_t D) {
    if (F.multiblank) return at::empty({N, 1 + D}, frames.options());
    return label_slots(frames.numel(), frames).view(frames.sizes());
}

// Loss from (N,T,U,V+D) TDT or (N,T,U,V) multi-blank logits, float32 or bfloat16: (costs (N), lse (N,T,U,2) or
// (N,T,U), grads (N,T,U,2+D) or empty), all float32.  No host sync.
template <const Lattice &F>
std::tuple<at::Tensor, at::Tensor, at::Tensor> lattice_forward(const at::Tensor &xs, const at::Tensor &ys,
                                                               const at::Tensor &xn, const at::Tensor &yn,
                                                               const std::vector<int> &durations, double sigma,
                                                               int blank, bool want_grads) {
    check4(xs, ys, xn, yn, true);
    check_batch4(xs, xn, yn);
    const int64_t N = xs.size(0), T = xs.size(1), U = xs.size(2), D = (int64_t)durations.size();
    check_arg(ys, Dt::I32, xs, {N, U - 1}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs");
    const int64_t V = lattice_tokens(F, xs.size(3), D, blank, F.row_cell);
    const c10::cuda::CUDAGuard guard(xs.device());
    const auto f32 = xs.options().dtype(at::kFloat);
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor lse = at::empty(lse_sizes(F, {N, T, U}), f32);
    at::Tensor pg = output(want_grads, {N, T, U, 2 + D}, f32);
    if (N == 0) return std::make_tuple(costs, lse, pg);
    at::Tensor ws = workspace(xs, F.workspace_bytes((int)N, (int)T, (int)U, (int)D));
    check_status(F.forward(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                           xn.data_ptr<int>(), yn.data_ptr<int>(), durations.data(), (int)D, (float)sigma,
                           costs.data_ptr<float>(), lse.data_ptr<float>(), want_grads ? pg.data_ptr<float>() : nullptr,
                           (int)N, (int)T, (int)U, (int)V, blank, elem_bytes(xs)));
    return std::make_tuple(costs, lse, pg);
}

// d loss / d logits (N,T,U,V+D) or (N,T,U,V), of the dtype of xs
template <const Lattice &F>
at::Tensor lattice_backward(const at::Tensor &xs, const at::Tensor &lse, const at::Tensor &grads, const at::Tensor &ys,
                            const std::vector<int> &durations, const at::Tensor &grad_out, int blank) {
    check_arg(xs, Dt::F32orBF16, xs, {kAny, kAny, kAny, kAny}, F.xs4);
    const int64_t N = xs.size(0), T = xs.size(1), U = xs.size(2), D = (int64_t)durations.size();
    const int64_t V = lattice_tokens(F, xs.size(3), D, blank, F.row_cell);
    check_arg(lse, Dt::F32, xs, lse_sizes(F, {N, T, U}), F.lse4);
    check_arg(grads, Dt::F32, xs, {N, T, U, 2 + D}, F.grads4);
    check_arg(ys, Dt::I32, xs, {N, U - 1}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs");
    check_arg(grad_out, Dt::F32, xs, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor out = at::empty_like(xs);
    if (N == 0) return out;
    check_status(F.backward(current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(), grads.data_ptr<float>(),
                            ys.data_ptr<int>(), durations.data(), (int)D, grad_out.data_ptr<float>(), out.data_ptr(),
                            (int)N, (int)T, (int)U, (int)V, blank, elem_bytes(xs)));
    return out;
}

// Loss from compact (STU,V+D) TDT or (STU,V) multi-blank logits in joint_pack's row order, float32 or bfloat16, labels
// (sum yn): (costs (N), lse (STU,2) or (STU), grads (STU,2+D) or empty, prefix (2N) int64 = {mem_pref, lab_pref} for
// the backward).  Shapes are validated as in rnnt_loss_compact: one 16-byte device->host copy, or none with hints
// (max_T, max_U > 0).
template <const Lattice &F>
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor>
lattice_compact_forward(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                        const std::vector<int> &durations, double sigma, int blank, bool want_grads, int max_T,
                        int max_U) {
    const auto [N, STU, W, bf16, guard] = compact_front(xs, ys, xn, yn, blank, true);
    const int64_t D = (int64_t)durations.size(), V = lattice_tokens(F, W, D, blank, F.row_row);
    void *stream = current_stream(xs);
    const auto f32 = xs.options().dtype(at::kFloat);
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor lse = at::empty(lse_sizes(F, {STU}), f32);
    at::Tensor pg = output(want_grads, {STU, 2 + D}, f32);
    at::Tensor prefix = at::empty({2 * N}, xs.options().dtype(at::kLong));
    if (N == 0) return std::make_tuple(costs, lse, pg, prefix);
    std::tie(max_T, max_U) = compact_bounds(stream, xs, ys, xn, yn, max_T, max_U, prefix.data_ptr<int64_t>());
    // a batch whose lengths are all 0: bounds of 1 (its lattices are invalid either way)
    max_T = std::max(max_T, 1);
    max_U = std::max(max_U, 1);
    at::Tensor ws = workspace(xs, F.compact_workspace_bytes(STU, (int)N, (int)D));
    check_status(F.compact_forward(stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                                   xn.data_ptr<int>(), yn.data_ptr<int>(), durations.data(), (int)D, (float)sigma,
                                   costs.data_ptr<float>(), lse.data_ptr<float>(),
                                   want_grads ? pg.data_ptr<float>() : nullptr, prefix.data_ptr<int64_t>(), nullptr,
                                   STU, (int)N, (int)V, blank, bf16 ? 2 : 4, max_T, max_U));
    return std::make_tuple(costs, lse, pg, prefix);
}

// d loss / d compact logits (STU,V+D) or (STU,V), of the dtype of xs
template <const Lattice &F>
at::Tensor lattice_compact_backward(const at::Tensor &xs, const at::Tensor &lse, const at::Tensor &grads,
                                    const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                                    const at::Tensor &prefix, const std::vector<int> &durations,
                                    const at::Tensor &grad_out, int blank) {
    check_arg(xs, Dt::F32orBF16, xs, {kAny, kAny}, F.xs2);
    const int64_t STU = xs.size(0), N = xn.numel(), D = (int64_t)durations.size();
    const int64_t V = lattice_tokens(F, xs.size(1), D, blank, F.row_row);
    if (F.multiblank)                                   // STU floats of any shape
        check_arg(lse, Dt::F32, xs, STU, F.lse2);
    else
        check_arg(lse, Dt::F32, xs, {STU, 2}, F.lse2);
    check_arg(grads, Dt::F32, xs, {STU, 2 + D}, F.grads2);
    TORCH_CHECK(is_arg(ys, Dt::I32, xs), "ys must be a contiguous Int tensor on the device of xs");
    const char *lengths = "xn and yn must be contiguous Int tensors of shape (N,) on the device of xs";
    check_arg(xn, Dt::I32, xs, N, lengths);
    check_arg(yn, Dt::I32, xs, N, lengths);
    check_arg(prefix, Dt::I64, xs, 2 * N, "prefix must be a contiguous Long tensor of shape (2N,) on the device of xs");
    check_arg(grad_out, Dt::F32, xs, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor out = at::empty_like(xs);
    if (N == 0 || STU == 0) return out;                 // empty tensors: nothing to write (and no data pointers)
    check_status(F.compact_backward(current_stream(xs), xs.data_ptr(), lse.data_ptr<float>(), grads.data_ptr<float>(),
                                    ys.data_ptr<int>(), yn.data_ptr<int>(), durations.data(), (int)D,
                                    prefix.data_ptr<int64_t>(), grad_out.data_ptr<float>(), out.data_ptr(), STU,
                                    (int)N, (int)V, blank, elem_bytes(xs)));
    return out;
}

// Viterbi alignment, dense (N,T,U,V+D) TDT or (N,T,U,V) multi-blank f32 or bf16 logits: (scores (N) f32, frames (N,U-1)
// i32, and TDT's label durations (N,U-1) i32 or multi-blank's blank counts (N,1+D) i32).  No host sync.
template <const Lattice &F>
std::tuple<at::Tensor, at::Tensor, at::Tensor> lattice_align_dense(const at::Tensor &xs, const at::Tensor &ys,
                                                                   const at::Tensor &xn, const at::Tensor &yn,
                                                                   const std::vector<int> &durations, double sigma,
                                                                   int blank) {
    check4(xs, ys, xn, yn, true);
    check_batch4(xs, xn, yn);
    const int64_t N = xs.size(0), T = xs.size(1), U = xs.size(2), D = (int64_t)durations.size();
    check_arg(ys, Dt::I32, xs, {N, U - 1}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs");
    const int64_t V = lattice_tokens(F, xs.size(3), D, blank, F.row_cell);
    const c10::cuda::CUDAGuard guard(xs.device());
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = label_slots(N * (U - 1), xs).view({N, U - 1});
    at::Tensor third = align_third(F, frames, N, D);
    if (N == 0) return std::make_tuple(scores, frames, third);
    at::Tensor ws = workspace(xs, F.align_workspace_bytes(N * T * U, (int)N, (int)D));
    check_status(F.align_dense(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                               xn.data_ptr<int>(), yn.data_ptr<int>(), durations.data(), (int)D, (float)sigma,
                               scores.data_ptr<float>(), frames.data_ptr<int>(), third.data_ptr<int>(), (int)N, (int)T,
                               (int)U, (int)V, blank, elem_bytes(xs)));
    return std::make_tuple(scores, frames, third);
}

// Viterbi alignment, compact (STU,V+D) TDT or (STU,V) multi-blank f32 or bf16 logits in joint_pack's row order, labels
// (sum yn): (scores (N) f32, frames (sum yn) i32, and TDT's label durations (sum yn) i32 or multi-blank's blank counts
// (N,1+D) i32).  The bounds are the hints when given (no host sync), else one 16-byte device->host copy.
template <const Lattice &F>
std::tuple<at::Tensor, at::Tensor, at::Tensor>
lattice_align_compact(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn, const at::Tensor &yn,
                      const std::vector<int> &durations, double sigma, int blank, int max_T, int max_U) {
    const auto [N, STU, W, bf16, guard] = compact_front(xs, ys, xn, yn, blank, true);
    const int64_t D = (int64_t)durations.size(), V = lattice_tokens(F, W, D, blank, F.row_row);
    void *stream = current_stream(xs);
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = label_slots(ys.numel(), xs);
    at::Tensor third = align_third(F, frames, N, D);
    if (N == 0) return std::make_tuple(scores, frames, third);
    std::tie(max_T, max_U) = compact_bounds(stream, xs, ys, xn, yn, max_T, max_U, nullptr);
    // a batch whose lengths are all 0: bounds of 1 (its lattices are invalid either way)
    max_T = std::max(max_T, 1);
    max_U = std::max(max_U, 1);
    at::Tensor ws = workspace(xs, F.align_workspace_bytes(STU, (int)N, (int)D));
    check_status(F.align_compact(stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                                 xn.data_ptr<int>(), yn.data_ptr<int>(), durations.data(), (int)D, (float)sigma,
                                 scores.data_ptr<float>(), frames.data_ptr<int>(), third.data_ptr<int>(), STU, (int)N,
                                 (int)V, blank, bf16 ? 2 : 4, max_T, max_U));
    return std::make_tuple(scores, frames, third);
}

// am (N,T,V) and lm (N,U,V): dtypes, then contiguity and device, then shapes; then ys, xn and yn
void check_simple_inputs(const at::Tensor &am, const at::Tensor &lm, const at::Tensor &ys, const at::Tensor &xn,
                         const at::Tensor &yn) {
    TORCH_CHECK(has_dtype(am, Dt::F32) && has_dtype(lm, Dt::F32),
                "am and lm must be float32 tensors (the simple loss does not take bfloat16)");
    TORCH_CHECK(am.is_contiguous() && lm.is_contiguous() && on_device(am, am) && on_device(lm, am),
                "am and lm must be contiguous CUDA tensors on one device");
    TORCH_CHECK(am.dim() == 3 && lm.dim() == 3 && lm.size(0) == am.size(0) && lm.size(2) == am.size(2),
                "am must be (N, T, V) and lm (N, U, V)");
    const int64_t N = am.size(0);
    check_arg(ys, Dt::I32, am, {N, lm.size(1) - 1}, "ys must be a contiguous Int tensor of shape (N, U-1) on the device of am");
    const char *lengths = "xn and yn must be contiguous Int tensors of shape (N,) on the device of am";
    check_arg(xn, Dt::I32, am, N, lengths);
    check_arg(yn, Dt::I32, am, N, lengths);
}

// the saved buffer of the simple loss: norm, oa, ol; with a smoothing scale also Ll, Am and log uni
int64_t simple_saved_len(int64_t N, int64_t T, int64_t U, int64_t V, bool smooth) {
    const int64_t base = N * T * U + N * T + N * U;
    return smooth ? base + N * U + N * T + V : base;
}

// simple loss from am (N,T,V) and lm (N,U,V), float32: (costs (N), saved (simple_saved_len), pair_grads (N,T,U,2) or
// empty, ranges (N,T) int32 or empty).  The pair gradients are computed when want_grads or prune_range > 0; the ranges
// when prune_range > 0.  lm_only_scale / am_only_scale: k2's smoothing (both 0: the plain simple loss).  No host sync.
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor>
rnnt_simple_forward(const at::Tensor &am, const at::Tensor &lm, const at::Tensor &ys, const at::Tensor &xn,
                    const at::Tensor &yn, int blank, bool want_grads, int prune_range, int lse_mode,
                    double lm_only_scale, double am_only_scale, int rnnt_type, double delay_penalty) {
    check_simple_inputs(am, lm, ys, xn, yn);
    const int64_t N = am.size(0), T = am.size(1), U = lm.size(1), V = am.size(2);
    check_blank(blank, V);
    TORCH_CHECK(prune_range == 0 || prune_range >= (rnnt_type == 0 ? 2 : 1),
                rnnt_type == 0 ? "prune_range must be an int >= 2" : "prune_range must be an int >= 1");
    const float sl = (float)lm_only_scale, sa = (float)am_only_scale;
    const bool smooth = sl != 0.0f || sa != 0.0f;
    const c10::cuda::CUDAGuard guard(am.device());
    const auto f32 = am.options().dtype(at::kFloat);
    const bool pairs = want_grads || prune_range > 0;
    at::Tensor costs = at::empty({N}, f32);
    at::Tensor saved = at::empty({simple_saved_len(N, T, U, V, smooth)}, f32);
    at::Tensor pg = output(pairs, {N, T, U, 2}, f32);
    at::Tensor ranges = at::empty({prune_range > 0 ? N : 0, prune_range > 0 ? T : 0}, am.options().dtype(at::kInt));
    // the constrained ranges score the blank edges before the fold: their gradient slots, kept for the ranges only
    at::Tensor raw = at::empty({rnnt_type == 2 && prune_range > 0 ? N * T * U : 0}, f32);
    float *rawp = raw.numel() ? raw.data_ptr<float>() : nullptr;
    if (N == 0) return std::make_tuple(costs, saved, pg, ranges);
    void *stream = current_stream(am);
    at::Tensor ws = workspace(am, smooth ? rnnt_b200_simple_smoothed_workspace_bytes((int)N, (int)T, (int)U, (int)V)
                                         : rnnt_b200_simple_workspace_bytes((int)N, (int)T, (int)U));
    check_status(rnnt_b200_simple_smoothed_forward_ex(
        stream, ws.data_ptr(), (size_t)ws.numel(), am.data_ptr<float>(), lm.data_ptr<float>(), ys.data_ptr<int>(),
        xn.data_ptr<int>(), yn.data_ptr<int>(), costs.data_ptr<float>(), saved.data_ptr<float>(),
        pairs ? pg.data_ptr<float>() : nullptr, (int)N, (int)T, (int)U, (int)V, blank, lse_mode, sl, sa, rnnt_type,
        (float)delay_penalty, rawp));
    if (prune_range > 0)
        check_status(rnnt_b200_prune_ranges_ex(stream, pg.data_ptr<float>(), rawp, xn.data_ptr<int>(), yn.data_ptr<int>(),
                                               (int)N, (int)T, (int)U, prune_range, rnnt_type, ranges.data_ptr<int>()));
    return std::make_tuple(costs, saved, pg, ranges);
}

// d sum_n grad_out[n] cost[n] / d (am, lm); the scales must be the forward's
std::tuple<at::Tensor, at::Tensor> rnnt_simple_backward(const at::Tensor &am, const at::Tensor &lm, const at::Tensor &ys,
                                                        const at::Tensor &xn, const at::Tensor &yn,
                                                        const at::Tensor &saved, const at::Tensor &pair_grads,
                                                        const at::Tensor &grad_out, int blank, double lm_only_scale,
                                                        double am_only_scale) {
    check_simple_inputs(am, lm, ys, xn, yn);
    const int64_t N = am.size(0), T = am.size(1), U = lm.size(1), V = am.size(2);
    const float sl = (float)lm_only_scale, sa = (float)am_only_scale;
    const bool smooth = sl != 0.0f || sa != 0.0f;
    check_arg(saved, Dt::F32, am, simple_saved_len(N, T, U, V, smooth),
              smooth ? "saved must be the smoothed simple forward's contiguous Float tensor on the device of am"
                     : "saved must be the simple forward's contiguous Float tensor on the device of am");
    check_arg(pair_grads, Dt::F32, am, N * T * U * 2,
              "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of am");
    check_arg(grad_out, Dt::F32, am, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    check_blank(blank, V);
    const c10::cuda::CUDAGuard guard(am.device());
    at::Tensor dam = at::empty_like(am), dlm = at::empty_like(lm);
    if (N == 0) return std::make_tuple(dam, dlm);
    at::Tensor ws = workspace(am, smooth ? rnnt_b200_simple_smoothed_workspace_bytes((int)N, (int)T, (int)U, (int)V) : 0);
    check_status(rnnt_b200_simple_smoothed_backward(current_stream(am), smooth ? ws.data_ptr() : nullptr,
                                                    (size_t)ws.numel(), am.data_ptr<float>(), lm.data_ptr<float>(),
                                                    ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(),
                                                    saved.data_ptr<float>(), pair_grads.data_ptr<float>(),
                                                    grad_out.data_ptr<float>(), dam.data_ptr<float>(),
                                                    dlm.data_ptr<float>(), (int)N, (int)T, (int)U, (int)V, blank, sl,
                                                    sa));
    return std::make_tuple(dam, dlm);
}

// prune ranges (N,T) int32 from pair gradients (N,T,U,2) of a loss call
at::Tensor rnnt_prune_ranges(const at::Tensor &pair_grads, const at::Tensor &xn, const at::Tensor &yn, int S,
                             int rnnt_type, const c10::optional<at::Tensor> &raw_blank) {
    check_arg(pair_grads, Dt::F32, pair_grads, {kAny, kAny, kAny, 2},
              "pair_grads must be a contiguous CUDA Float tensor of shape (N, T, U, 2)");
    const int64_t N = pair_grads.size(0), T = pair_grads.size(1), U = pair_grads.size(2);
    const char *lengths = "xn and yn must be contiguous Int tensors of shape (N,) on the device of pair_grads";
    check_arg(xn, Dt::I32, pair_grads, N, lengths);
    check_arg(yn, Dt::I32, pair_grads, N, lengths);
    TORCH_CHECK(rnnt_type >= 0 && rnnt_type <= 2, "rnnt_type must be 0, 1 or 2");
    TORCH_CHECK(S >= (rnnt_type == 0 ? 2 : 1),
                rnnt_type == 0 ? "prune_range must be an int >= 2" : "prune_range must be an int >= 1");
    const bool use_raw = rnnt_type == 2;
    TORCH_CHECK(!use_raw || raw_blank.has_value(), "rnnt_type 2 needs raw_blank");
    if (use_raw)
        check_arg(*raw_blank, Dt::F32, pair_grads, N * T * U,
                  "raw_blank must be a contiguous Float tensor of shape (N, T, U) on the device of pair_grads");
    const c10::cuda::CUDAGuard guard(pair_grads.device());
    at::Tensor ranges = at::empty({N, T}, pair_grads.options().dtype(at::kInt));
    if (N == 0) return ranges;
    check_status(rnnt_b200_prune_ranges_ex(current_stream(pair_grads), pair_grads.data_ptr<float>(),
                                           use_raw ? raw_blank->data_ptr<float>() : nullptr, xn.data_ptr<int>(),
                                           yn.data_ptr<int>(), (int)N, (int)T, (int)U, S, rnnt_type,
                                           ranges.data_ptr<int>()));
    return ranges;
}

// compact packing of the joint input: (x (STU,H), mem_pref (N) int64).  stu < 0: STU is read back from the device
// (one 16-byte copy); stu >= 0: trusted, no host sync.
std::tuple<at::Tensor, at::Tensor> rnnt_joint_pack(const at::Tensor &f, const at::Tensor &g, const at::Tensor &lf,
                                                   const at::Tensor &lg, int64_t stu) {
    // contiguity, then dtypes, then device, each for all four
    TORCH_CHECK(f.is_contiguous() && g.is_contiguous() && lf.is_contiguous() && lg.is_contiguous(), "inputs must be contiguous");
    TORCH_CHECK(has_dtype(f, Dt::F32) && has_dtype(g, Dt::F32), "f and g must be Float tensors");
    TORCH_CHECK(has_dtype(lf, Dt::I32) && has_dtype(lg, Dt::I32), "lf and lg must be Int tensors");
    TORCH_CHECK(on_device(f, f) && on_device(g, f) && on_device(lf, f) && on_device(lg, f),
                "f, g, lf, lg must be on the same CUDA device");
    TORCH_CHECK(f.dim() == 3 && g.dim() == 3 && f.size(0) == g.size(0) && f.size(2) == g.size(2),
                "f must be (N, T, H) and g (N, U+1, H)");
    const int64_t N = f.size(0), T = f.size(1), U1 = g.size(1), H = f.size(2);
    TORCH_CHECK(lf.numel() == N && lg.numel() == N, "lf and lg must have N elements");
    const c10::cuda::CUDAGuard guard(f.device());
    void *stream = current_stream(f);
    at::Tensor scratch = at::empty({2 * std::max<int64_t>(N, 1)}, f.options().dtype(at::kLong));
    if (N == 0) return std::make_tuple(at::empty({0, H}, f.options()), scratch);
    if (stu < 0) {
        at::Tensor totals = at::empty({4}, f.options().dtype(at::kInt));
        check_status(rnnt_b200_joint_pack(stream, nullptr, nullptr, lf.data_ptr<int>(), lg.data_ptr<int>(),
                                          scratch.data_ptr<int64_t>(), totals.data_ptr<int>(), nullptr, (int)N, (int)T,
                                          (int)U1, (int)H, 0));
        at::Tensor h = totals.cpu();
        const int *t = h.data_ptr<int>();
        TORCH_CHECK(t[2] <= T && t[3] <= U1, "lf / lg exceed the shapes of f / g");
        stu = t[0];
    }
    at::Tensor x = at::empty({stu, H}, f.options());
    check_status(rnnt_b200_joint_pack(stream, f.data_ptr<float>(), g.data_ptr<float>(), lf.data_ptr<int>(),
                                      lg.data_ptr<int>(), scratch.data_ptr<int64_t>(), nullptr, x.data_ptr<float>(), (int)N,
                                      (int)T, (int)U1, (int)H, stu));
    return std::make_tuple(x, scratch.narrow(0, 0, N));
}

std::tuple<at::Tensor, at::Tensor> rnnt_joint_pack_backward(const at::Tensor &dx, const at::Tensor &lf,
                                                            const at::Tensor &lg, const at::Tensor &mem_pref,
                                                            int64_t T, int64_t U1) {
    check_arg(dx, Dt::F32, dx, {kAny, kAny}, "dx must be a contiguous CUDA Float tensor of shape (STU, H)");
    TORCH_CHECK(is_arg(mem_pref, Dt::I64, dx), "mem_pref must be a contiguous Long tensor on the device of dx");
    const int64_t N = mem_pref.numel(), H = dx.size(1);
    TORCH_CHECK(lf.numel() == N && lg.numel() == N && lf.is_contiguous() && lg.is_contiguous() &&
                    has_dtype(lf, Dt::I32) && has_dtype(lg, Dt::I32),
                "lf and lg must be contiguous Int tensors with N elements");
    TORCH_CHECK(on_device(lf, dx) && on_device(lg, dx), "lf and lg must be on the device of dx");
    const c10::cuda::CUDAGuard guard(dx.device());
    at::Tensor df = at::empty({N, T, H}, dx.options()), dg = at::empty({N, U1, H}, dx.options());
    check_status(rnnt_b200_joint_pack_backward(current_stream(dx), dx.data_ptr<float>(), lf.data_ptr<int>(),
                                               lg.data_ptr<int>(), mem_pref.data_ptr<int64_t>(), df.data_ptr<float>(),
                                               dg.data_ptr<float>(), (int)N, (int)T, (int)U1, (int)H));
    return std::make_tuple(df, dg);
}

at::Tensor rnnt_gather_backward(const at::Tensor &pair_grads, const at::Tensor &ys, const at::Tensor &grad_out,
                                int64_t V, int blank, bool accumulate, const c10::optional<at::Tensor> &yn) {
    check_arg(pair_grads, Dt::F32, pair_grads, {kAny, kAny, kAny, 2},
              "pair_grads must be a contiguous CUDA Float tensor of shape (N, T, U, 2)");
    TORCH_CHECK(is_arg(ys, Dt::I32, pair_grads), "ys must be a contiguous Int tensor on the device of pair_grads");
    const int64_t N = pair_grads.size(0), T = pair_grads.size(1), U = pair_grads.size(2);
    check_arg(grad_out, Dt::F32, pair_grads, N, "grad_out must be a contiguous Float tensor of shape (N,)");
    TORCH_CHECK(has_sizes(ys, {N, U - 1}), "ys shape (N, U-1) mismatched");
    check_blank(blank, V);
    const int *ynp = optional_arg<int>(yn, Dt::I32, pair_grads, N,
                                       "yn must be a contiguous Int tensor of shape (N,) on the device of pair_grads");
    const c10::cuda::CUDAGuard guard(pair_grads.device());
    at::Tensor out = at::empty({N, T, U, V}, pair_grads.options());
    check_status(rnnt_b200_gather_backward(current_stream(pair_grads), pair_grads.data_ptr<float>(),
                                           ys.data_ptr<int>(), grad_out.data_ptr<float>(), out.data_ptr<float>(),
                                           (int)N, (int)T, (int)U, (int)V, blank, accumulate ? 1 : 0, ynp));
    return out;
}

// Viterbi alignment, dense (N,T,U,V) f32 or bf16 log-probs: (scores (N) f32, frames (N,U-1) i32).  No host sync.
std::tuple<at::Tensor, at::Tensor> rnnt_align_dense(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                                    const at::Tensor &yn, int blank) {
    const auto [N, T, U, V, bf16, guard] = dense_front(xs, ys, xn, yn, true);
    check_blank(blank, V);
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = at::empty({N, U - 1}, xs.options().dtype(at::kInt));
    if (N == 0) return std::make_tuple(scores, frames);
    at::Tensor ws = workspace(xs, rnnt_b200_align_workspace_bytes(N * T * U, (int)N, (int)T, (int)U));
    check_status(rnnt_b200_align_dense(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(),
                                       ys.data_ptr<int>(), xn.data_ptr<int>(), yn.data_ptr<int>(),
                                       scores.data_ptr<float>(), frames.data_ptr<int>(), (int)N, (int)T, (int)U, (int)V,
                                       blank, bf16 ? 2 : 4));
    return std::make_tuple(scores, frames);
}

// Viterbi alignment, compact (STU,V) f32 or bf16 log-probs: (scores (N) f32, frames (sum yn) i32).  The bounds are
// the hints when given (no host sync), else one 16-byte device->host copy, as in rnnt_loss_compact.
std::tuple<at::Tensor, at::Tensor> rnnt_align_compact(const at::Tensor &xs, const at::Tensor &ys, const at::Tensor &xn,
                                                      const at::Tensor &yn, int blank, int max_T, int max_U) {
    const auto [N, STU, V, bf16, guard] = compact_front(xs, ys, xn, yn, blank, true);
    void *stream = current_stream(xs);
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = at::empty({ys.numel()}, xs.options().dtype(at::kInt));
    if (N == 0) return std::make_tuple(scores, frames);
    std::tie(max_T, max_U) = compact_bounds(stream, xs, ys, xn, yn, max_T, max_U, nullptr);
    max_T = std::max(max_T, 1);              // lengths of 0 or less: the lattice is outside any bounds (score NaN)
    max_U = std::max(max_U, 1);
    at::Tensor ws = workspace(xs, rnnt_b200_align_workspace_bytes(STU, (int)N, max_T, max_U));
    check_status(rnnt_b200_align_compact(stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                                         xn.data_ptr<int>(), yn.data_ptr<int>(), scores.data_ptr<float>(),
                                         frames.data_ptr<int>(), STU, (int)N, (int)V, blank, bf16 ? 2 : 4, max_T,
                                         max_U));
    return std::make_tuple(scores, frames);
}

// Viterbi alignment from dense (N,T,U,V) f32 or bf16 logits on k2's lattices (rnnt_type 0, 1, 2, delay_penalty):
// (scores (N) f32, frames (N,U-1) i32).  No host sync.
std::tuple<at::Tensor, at::Tensor> rnnt_align_logits_dense(const at::Tensor &xs, const at::Tensor &ys,
                                                           const at::Tensor &xn, const at::Tensor &yn, int blank,
                                                           int rnnt_type, double delay_penalty, bool hat) {
    const auto [N, T, U, V, bf16, guard] = dense_front(xs, ys, xn, yn, true);
    check_blank(blank, V);
    check_hat(hat, V);
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = label_slots(N * (U - 1), xs).view({N, U - 1});
    if (N == 0) return std::make_tuple(scores, frames);
    at::Tensor ws = workspace(xs, rnnt_b200_align_logits_workspace_bytes(N * T * U, (int)N, (int)T, (int)U));
    const auto align = hat ? rnnt_b200_align_logits_hat_dense : rnnt_b200_align_logits_dense;
    check_status(align(current_stream(xs), ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(),
                       xn.data_ptr<int>(), yn.data_ptr<int>(), scores.data_ptr<float>(), frames.data_ptr<int>(),
                       (int)N, (int)T, (int)U, (int)V, blank, bf16 ? 2 : 4, rnnt_type, (float)delay_penalty));
    return std::make_tuple(scores, frames);
}

// Viterbi alignment from compact (STU,V) f32 or bf16 logits in joint_pack's row order (regular lattice): (scores (N)
// f32, frames (sum yn) i32).  The bounds are the hints when given (no host sync), else one 16-byte device->host copy.
std::tuple<at::Tensor, at::Tensor> rnnt_align_logits_compact(const at::Tensor &xs, const at::Tensor &ys,
                                                             const at::Tensor &xn, const at::Tensor &yn, int blank,
                                                             int max_T, int max_U, bool hat) {
    const auto [N, STU, V, bf16, guard] = compact_front(xs, ys, xn, yn, blank, true);
    check_hat(hat, V);
    void *stream = current_stream(xs);
    at::Tensor scores = at::empty({N}, xs.options().dtype(at::kFloat));
    at::Tensor frames = label_slots(ys.numel(), xs);
    if (N == 0) return std::make_tuple(scores, frames);
    std::tie(max_T, max_U) = compact_bounds(stream, xs, ys, xn, yn, max_T, max_U, nullptr);
    max_T = std::max(max_T, 1);              // lengths of 0 or less: the lattice is outside any bounds (score NaN)
    max_U = std::max(max_U, 1);
    at::Tensor ws = workspace(xs, rnnt_b200_align_logits_workspace_bytes(STU, (int)N, max_T, max_U));
    const auto align = hat ? rnnt_b200_align_logits_hat_compact : rnnt_b200_align_logits_compact;
    check_status(align(stream, ws.data_ptr(), (size_t)ws.numel(), xs.data_ptr(), ys.data_ptr<int>(), xn.data_ptr<int>(),
                       yn.data_ptr<int>(), scores.data_ptr<float>(), frames.data_ptr<int>(), STU, (int)N, (int)V,
                       blank, bf16 ? 2 : 4, max_T, max_U));
    return std::make_tuple(scores, frames);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    namespace py = pybind11;
    m.def("rnnt_loss", &rnnt_loss, "H100 RNN-Transducer loss (forward and gradients).", py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0);
    m.def("rnnt_loss_compact", &rnnt_loss_compact, "H100 RNN-Transducer loss in compact layout.", py::arg("xs"),
          py::arg("ys"), py::arg("xn"), py::arg("yn"), py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0,
          py::arg("required_grad") = true, py::arg("max_T") = 0, py::arg("max_U") = 0);
    m.def("rnnt_loss_compact_backward", &rnnt_loss_compact_backward,
          "H100 RNN-Transducer loss backward for compact layout", py::arg("grad_costs"), py::arg("grad_xs"),
          py::arg("cumSum"), py::arg("loc"), py::arg("V"), py::arg("blank") = 0);
    m.def("rnnt_loss_dense", &rnnt_loss_dense, py::arg("xs"), py::arg("ys"), py::arg("xn"), py::arg("yn"),
          py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0, py::arg("grad_scale") = py::none(),
          py::arg("want_grads") = true, py::arg("lse_mode") = 0);
    m.def("rnnt_loss_fused", &rnnt_loss_fused, py::arg("xs"), py::arg("ys"), py::arg("xn"), py::arg("yn"),
          py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0, py::arg("grad_scale") = py::none(),
          py::arg("want_grads") = true, py::arg("lse_mode") = 0);
    m.def("rnnt_rescale_", &rnnt_rescale_, py::arg("grads"), py::arg("grad_out"), py::arg("applied") = py::none());
    m.def("rnnt_logits_forward", &rnnt_logits_forward, py::arg("xs"), py::arg("ys"), py::arg("xn"), py::arg("yn"),
          py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0, py::arg("want_grads") = true, py::arg("lse_mode") = 0,
          py::arg("rnnt_type") = 0, py::arg("delay_penalty") = 0.0, py::arg("hat") = false);
    m.def("rnnt_logits_backward", &rnnt_logits_backward, py::arg("xs"), py::arg("lse"), py::arg("pair_grads"),
          py::arg("ys"), py::arg("grad_out"), py::arg("blank") = 0, py::arg("hat") = false);
    m.def("rnnt_logits_compact_forward", &rnnt_logits_compact_forward, py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0, py::arg("want_grads") = true,
          py::arg("lse_mode") = 0, py::arg("max_T") = 0, py::arg("max_U") = 0, py::arg("hat") = false);
    m.def("rnnt_logits_compact_backward", &rnnt_logits_compact_backward, py::arg("xs"), py::arg("lse"),
          py::arg("pair_grads"), py::arg("ys"), py::arg("xn"), py::arg("yn"), py::arg("prefix"), py::arg("grad_out"),
          py::arg("blank") = 0, py::arg("hat") = false);
    m.def("rnnt_logits_pruned_forward", &rnnt_logits_pruned_forward, py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("ranges"), py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0,
          py::arg("want_grads") = true, py::arg("lse_mode") = 0, py::arg("rnnt_type") = 0,
          py::arg("delay_penalty") = 0.0, py::arg("hat") = false);
    m.def("rnnt_logits_pruned_backward", &rnnt_logits_pruned_backward, py::arg("xs"), py::arg("lse"),
          py::arg("pair_grads"), py::arg("ys"), py::arg("ranges"), py::arg("grad_out"), py::arg("blank") = 0,
          py::arg("hat") = false);
    m.def("rnnt_tdt_forward", &lattice_forward<kTdt>, py::arg("xs"), py::arg("ys"), py::arg("xn"), py::arg("yn"),
          py::arg("durations"), py::arg("sigma") = 0.0, py::arg("blank") = 0, py::arg("want_grads") = true);
    m.def("rnnt_tdt_backward", &lattice_backward<kTdt>, py::arg("xs"), py::arg("lse"), py::arg("grads"), py::arg("ys"),
          py::arg("durations"), py::arg("grad_out"), py::arg("blank") = 0);
    m.def("rnnt_tdt_compact_forward", &lattice_compact_forward<kTdt>, py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("durations"), py::arg("sigma"), py::arg("blank"), py::arg("want_grads"),
          py::arg("max_T") = 0, py::arg("max_U") = 0);
    m.def("rnnt_tdt_compact_backward", &lattice_compact_backward<kTdt>, py::arg("xs"), py::arg("lse"), py::arg("grads"),
          py::arg("ys"), py::arg("xn"), py::arg("yn"), py::arg("prefix"), py::arg("durations"), py::arg("grad_out"),
          py::arg("blank"));
    m.def("rnnt_multiblank_forward", &lattice_forward<kMultiblank>, py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("big_blank_durations"), py::arg("sigma"), py::arg("blank"), py::arg("want_grads") = true);
    m.def("rnnt_multiblank_backward", &lattice_backward<kMultiblank>, py::arg("xs"), py::arg("lse"), py::arg("grads"),
          py::arg("ys"), py::arg("big_blank_durations"), py::arg("grad_out"), py::arg("blank"));
    m.def("rnnt_multiblank_compact_forward", &lattice_compact_forward<kMultiblank>, py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("big_blank_durations"), py::arg("sigma"), py::arg("blank"),
          py::arg("want_grads"), py::arg("max_T") = 0, py::arg("max_U") = 0);
    m.def("rnnt_multiblank_compact_backward", &lattice_compact_backward<kMultiblank>, py::arg("xs"), py::arg("lse"),
          py::arg("grads"), py::arg("ys"), py::arg("xn"), py::arg("yn"), py::arg("prefix"),
          py::arg("big_blank_durations"), py::arg("grad_out"), py::arg("blank"));
    m.def("rnnt_tdt_align_dense", &lattice_align_dense<kTdt>,
          "Viterbi forced alignment on the TDT lattice, dense layout.", py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("durations"), py::arg("sigma") = 0.0, py::arg("blank") = 0);
    m.def("rnnt_tdt_align_compact", &lattice_align_compact<kTdt>,
          "Viterbi forced alignment on the TDT lattice, compact layout.", py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("durations"), py::arg("sigma") = 0.0, py::arg("blank") = 0, py::arg("max_T") = 0,
          py::arg("max_U") = 0);
    m.def("rnnt_multiblank_align_dense", &lattice_align_dense<kMultiblank>,
          "Viterbi forced alignment on the multi-blank lattice, dense layout.", py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("big_blank_durations"), py::arg("sigma"), py::arg("blank"));
    m.def("rnnt_multiblank_align_compact", &lattice_align_compact<kMultiblank>,
          "Viterbi forced alignment on the multi-blank lattice, compact layout.", py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("big_blank_durations"), py::arg("sigma"), py::arg("blank"),
          py::arg("max_T") = 0, py::arg("max_U") = 0);
    m.def("rnnt_simple_forward", &rnnt_simple_forward, py::arg("am"), py::arg("lm"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("blank") = 0, py::arg("want_grads") = true, py::arg("prune_range") = 0,
          py::arg("lse_mode") = 0, py::arg("lm_only_scale") = 0.0, py::arg("am_only_scale") = 0.0,
          py::arg("rnnt_type") = 0, py::arg("delay_penalty") = 0.0);
    m.def("rnnt_simple_backward", &rnnt_simple_backward, py::arg("am"), py::arg("lm"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("saved"), py::arg("pair_grads"), py::arg("grad_out"), py::arg("blank") = 0,
          py::arg("lm_only_scale") = 0.0, py::arg("am_only_scale") = 0.0);
    m.def("rnnt_prune_ranges", &rnnt_prune_ranges, py::arg("pair_grads"), py::arg("xn"), py::arg("yn"), py::arg("S"),
          py::arg("rnnt_type") = 0, py::arg("raw_blank") = py::none());
    m.def("rnnt_joint_pack", &rnnt_joint_pack, py::arg("f"), py::arg("g"), py::arg("lf"), py::arg("lg"), py::arg("stu") = -1);
    m.def("rnnt_joint_pack_backward", &rnnt_joint_pack_backward, py::arg("dx"), py::arg("lf"), py::arg("lg"),
          py::arg("mem_pref"), py::arg("T"), py::arg("U1"));
    m.def("rnnt_gather_forward", &rnnt_gather_forward, py::arg("xs"), py::arg("ys"), py::arg("xn"), py::arg("yn"),
          py::arg("blank") = 0, py::arg("fastemit_lambda") = 0.0, py::arg("want_grads") = true,
          py::arg("lse_mode") = 0);
    m.def("rnnt_gather_backward", &rnnt_gather_backward, py::arg("pair_grads"), py::arg("ys"), py::arg("grad_out"),
          py::arg("V"), py::arg("blank") = 0, py::arg("accumulate") = false, py::arg("yn") = py::none());
    m.def("rnnt_align_dense", &rnnt_align_dense, "Viterbi forced alignment, dense layout.", py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("blank") = 0);
    m.def("rnnt_align_compact", &rnnt_align_compact, "Viterbi forced alignment, compact layout.", py::arg("xs"),
          py::arg("ys"), py::arg("xn"), py::arg("yn"), py::arg("blank") = 0, py::arg("max_T") = 0,
          py::arg("max_U") = 0);
    m.def("rnnt_align_logits_dense", &rnnt_align_logits_dense,
          "Viterbi forced alignment from logits on k2's lattices, dense layout.", py::arg("xs"), py::arg("ys"),
          py::arg("xn"), py::arg("yn"), py::arg("blank") = 0, py::arg("rnnt_type") = 0, py::arg("delay_penalty") = 0.0,
          py::arg("hat") = false);
    m.def("rnnt_align_logits_compact", &rnnt_align_logits_compact,
          "Viterbi forced alignment from logits, compact layout.", py::arg("xs"), py::arg("ys"), py::arg("xn"),
          py::arg("yn"), py::arg("blank") = 0, py::arg("max_T") = 0, py::arg("max_U") = 0, py::arg("hat") = false);
    m.def("set_lse_mode", [](int mode) { rnnt_b200_set_lse_mode(mode); }, py::arg("mode"));
    m.def("get_lse_mode", []() { return rnnt_b200_get_lse_mode(); });
    m.def("launch_count", []() { return rnnt_b200_launch_count(); });
    m.def("version", []() { return std::string(rnnt_b200_version()); });
}
