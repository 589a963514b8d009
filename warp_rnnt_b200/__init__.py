"""warp_rnnt_b200 -- H100-native RNN-Transducer loss, drop-in for 1ytic/warp-rnnt's
``warp_rnnt.rnnt_loss`` (reference: the reference's pytorch_binding/warp_rnnt/__init__.py).

Same public surface as the reference module (``__init__.py:9-143``):

    rnnt_loss(log_probs, labels, frames_lengths, labels_lengths, average_frames=False,
              reduction='none', blank=0, gather=False, fastemit_lambda=0.0, compact=False)
    RNNTLoss, RNNTLossCompact (autograd Functions), __version__, and the operator module ``_C``
    (rnnt_loss / rnnt_loss_compact / rnnt_loss_compact_backward, same kwargs and error strings).

Host code here is plumbing only (argument handling, autograd wiring); all arithmetic runs in the
hand-written sm_90a kernels of ``lib/librnnt_b200.so`` through ``lib/_C.so``.  There is no CPU or
eager-PyTorch fallback: importing this package without the built extension raises ImportError.
"""
import contextlib
import importlib.machinery
import importlib.util
import math
import os
import sys
import threading

import torch

__version__ = "0.1.0"

_HERE = os.path.dirname(os.path.abspath(__file__))
_EXT_PATH = os.path.join(_HERE, "lib", "_C.so")
_LIB_PATH = os.path.join(_HERE, "lib", "librnnt_b200.so")


def _load_ext():
    # Stale binaries must not load silently: lib/sources.sha256 records the content hash of the sources the two
    # artefacts were built from; on a mismatch (edited sources, a pull) they are rebuilt -- or, with
    # RNNT_B200_NO_AUTOBUILD=1, the import fails.
    from . import build as _build
    if not _build.up_to_date():
        if os.environ.get("RNNT_B200_NO_AUTOBUILD") == "1":
            raise ImportError(
                "warp_rnnt_b200: the CUDA extension is missing or older than its sources (%s). "
                "Run `python -m warp_rnnt_b200.build`; there is no CPU fallback." % _EXT_PATH)
        _build.build_all()                   # builds the CUDA extension itself (nvcc + g++)
    name = __name__ + "._C"
    loader = importlib.machinery.ExtensionFileLoader(name, _EXT_PATH)
    spec = importlib.util.spec_from_file_location(name, _EXT_PATH, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


_C = _load_ext()
core = _C

LSE_AUTO, LSE_EXACT, LSE_FAST = 0, 1, 2


def set_lse_mode(mode):
    """'auto' | 'exact' | 'fast' (see include/rnnt_b200.h rnntLseMode_t).  'exact' (= 'auto', the
    default) reproduces the reference kernels' alpha/beta/cost/gradient bits; 'fast' shortens the
    wavefront's dependent chain at the price of fp32-noise-level differences (<= ~1e-4 on gradients)."""
    _C.set_lse_mode({"auto": 0, "exact": 1, "fast": 2}[mode] if isinstance(mode, str) else int(mode))


class RNNTLoss(torch.autograd.Function):
    """Dense loss, ONE kernel launch per step.  Reference: ``RNNTLoss`` (__init__.py:9-24).

    Like the reference, forward produces the dense gradient; unlike it, the python-level reduction
    (average_frames, 'sum' / 'mean', __init__.py:132-143) is part of this Function: the per-sample weights
    ``weights[n]`` (1/N, 1/frames, ...) go into the kernel as ``grad_scale``, the kernel returns
    ``sum_n weights[n] * cost[n]`` itself (``reduce=True``) and the gradient it wrote already is
    d(loss)/d(log_probs).  Backward then only has to compare the upstream gradient with what was multiplied
    in (``rnnt_rescale_``: a tiny launch that touches no gradient memory when they agree -- the usual
    ``loss.backward()``) instead of the reference's dense ``mul_`` (two more passes over (N,T,U,V)).

    With ``blank == -1`` the input is the gathered (N,T,U,2) layout of the reference's operator boundary
    (binding.cpp:81-90); weights / reduce are not supported there."""

    @staticmethod
    def forward(ctx, log_probs, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0,
                weights=None, reduce=False):
        need = ctx.needs_input_grad[0]
        ctx.need = need
        if blank == -1:
            assert weights is None and not reduce
            costs, grads = _C.rnnt_loss_dense(log_probs, labels, frames_lengths, labels_lengths, -1,
                                              fastemit_lambda, None, need, 0)
            ctx.grads = grads if need else None
            return costs
        costs, grads, loss = _C.rnnt_loss_fused(log_probs, labels, frames_lengths, labels_lengths, blank,
                                                fastemit_lambda, weights, need, 0)
        ctx.grads = grads if need else None
        if reduce:
            return loss[0]
        return costs if weights is None else costs * weights

    @staticmethod
    def backward(ctx, grads_output):
        if not ctx.need:
            return None, None, None, None, None, None, None, None
        g, ctx.grads = ctx.grads, None       # hand the buffer over: autograd can then adopt it as .grad without a copy
        if g is None:
            raise RuntimeError("RNNTLoss: backward called a second time, but the gradient buffer produced by forward "
                               "has already been handed to autograd (run forward again)")
        go = grads_output.detach().reshape(-1).to(torch.float32).contiguous()
        _C.rnnt_rescale_(g, go, None)        # in place, like the reference's mul_ (__init__.py:23); no-op when go == 1
        return g, None, None, None, None, None, None, None


class RNNTLossGather(torch.autograd.Function):
    """``gather=True``: the reference's memory-saving mode (__init__.py:118-128).  Forward keeps the gradient in
    its (N,T,U,2) [blank,label] form -- the log-prob gather runs inside the forward kernel, without the int64
    index tensor -- and backward emits the dense (N,T,U,V) tensor once, already scaled by grad_output (replaces
    mul_ + GatherBackward's zeros + scatter_add_).  A label equal to ``blank`` adds both gradients, as
    torch.gather's backward does."""

    @staticmethod
    def forward(ctx, log_probs, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0):
        need = ctx.needs_input_grad[0]
        costs, pg = _C.rnnt_gather_forward(log_probs, labels, frames_lengths, labels_lengths, blank,
                                           fastemit_lambda, need, 0)
        ctx.grads = pg if need else None
        ctx.labels = labels
        ctx.yn = labels_lengths
        ctx.V = log_probs.size(3)
        ctx.blank = blank
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        if ctx.grads is None:
            return None, None, None, None, None, None
        go = grads_output.contiguous().to(ctx.grads.dtype)
        g = _C.rnnt_gather_backward(ctx.grads, ctx.labels, go, ctx.V, ctx.blank, True, ctx.yn)
        return g, None, None, None, None, None


class RNNTLossFromLogits(torch.autograd.Function):
    """Loss straight from un-normalised joint-network logits: ``log_softmax`` fused into the loss (SURVEY.md 8(f)1).

    The reference needs log-softmaxed input (README.md:59; its benchmark times ``F.log_softmax`` with the loss,
    benchmark.py:65): seven dense passes over (N,T,U,V) per step.  Here forward reads the logits once (per-cell
    normaliser + the two log-probs the recurrence needs) and keeps a (N,T,U,2) gradient; backward reads them once more
    and writes d loss / d LOGITS, applying log_softmax's backward on the fly: three dense passes.  float32 or bfloat16
    logits; the gradient has the logits' dtype, costs are float32.  ``hat``: the HAT normalisation in place of
    log_softmax (``rnnt_loss_from_logits(use_hat_loss=True)``)."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0, rnnt_type=0,
                delay_penalty=0.0, hat=False):
        need = ctx.needs_input_grad[0]
        costs, lse, pg = _C.rnnt_logits_forward(logits, labels, frames_lengths, labels_lengths, blank,
                                                fastemit_lambda, need, 0, rnnt_type, delay_penalty, hat)
        if need:
            ctx.save_for_backward(logits, lse, pg, labels)
            ctx.blank = blank
            ctx.hat = hat
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_logits_backward(logits, lse, pg, labels, go, ctx.blank, ctx.hat)
        return g, None, None, None, None, None, None, None, None


class RNNTLossFromLogitsCompact(torch.autograd.Function):
    """``RNNTLossFromLogits`` on compact (STU,V) logits in ``joint_pack``'s row order: a packed joint network feeds
    the fused loss without padding.  Forward keeps lse (4 bytes per row), the (STU,2) pair gradients (8 bytes per row)
    and the compact prefix sums (16 bytes per lattice); backward writes d loss / d logits, of the logits' dtype.  Inside
    ``compact_hints`` the forward has no host sync (CUDA-graph capturable), as ``rnnt_loss(compact=True)``.  ``hat``:
    the HAT normalisation in place of log_softmax."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0, hat=False):
        need = ctx.needs_input_grad[0]
        hints = _hints()
        costs, lse, pg, prefix = _C.rnnt_logits_compact_forward(logits, labels, frames_lengths, labels_lengths, blank,
                                                                fastemit_lambda, need, 0, hints[0], hints[1], hat)
        if need:
            ctx.save_for_backward(logits, lse, pg, labels, frames_lengths, labels_lengths, prefix)
            ctx.blank = blank
            ctx.hat = hat
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels, xn, yn, prefix = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_logits_compact_backward(logits, lse, pg, labels, xn, yn, prefix, go, ctx.blank, ctx.hat)
        return g, None, None, None, None, None, None


def _reduce(costs, frames_lengths, average_frames, reduction):
    """The float32 costs of a loss call divided by the frame counts when ``average_frames``, then summed or averaged
    for ``reduction`` 'sum' or 'mean' ('none' and None keep them)."""
    if average_frames:
        costs = costs / frames_lengths.to(costs.dtype)      # float32: bf16 would round frame counts (601 -> 600)
    if reduction == "sum":
        return costs.sum()
    if reduction == "mean":
        return costs.mean()
    return costs


_RNNT_TYPES = {"regular": 0, "modified": 1, "constrained": 2}


def _path_type(fn, rnnt_type, delay_penalty, fastemit_lambda=0.0, compact=False):
    """k2's ``rnnt_type`` and ``delay_penalty`` checked on the host: (type id, penalty), or ValueError."""
    if not isinstance(rnnt_type, str) or rnnt_type not in _RNNT_TYPES:
        raise ValueError("%s: rnnt_type must be 'regular', 'modified' or 'constrained', got %r" % (fn, rnnt_type))
    if isinstance(delay_penalty, bool) or not isinstance(delay_penalty, (int, float)) \
            or not math.isfinite(delay_penalty) or delay_penalty < 0:
        raise ValueError("%s: delay_penalty must be a finite number >= 0, got %r" % (fn, delay_penalty))
    if rnnt_type != "regular" and fastemit_lambda != 0:
        raise ValueError("%s: fastemit_lambda is only offered with rnnt_type='regular', got %r with %r"
                         % (fn, fastemit_lambda, rnnt_type))
    if compact and (rnnt_type != "regular" or delay_penalty != 0):
        raise ValueError("%s: compact=True takes rnnt_type='regular' and delay_penalty=0 only" % fn)
    return _RNNT_TYPES[rnnt_type], float(delay_penalty)


def _use_hat(fn, use_hat_loss, logits):
    """k2's ``use_hat_loss`` checked on the host: a bool, and V >= 2 when set (the labels need a column besides the
    blank); ValueError otherwise."""
    if not isinstance(use_hat_loss, bool):
        raise ValueError("%s: use_hat_loss must be a bool, got %r" % (fn, use_hat_loss))
    if use_hat_loss and logits.dim() > 0 and logits.size(-1) < 2:
        raise ValueError("%s: use_hat_loss=True needs V >= 2, got V = %d" % (fn, logits.size(-1)))
    return use_hat_loss


def rnnt_loss_from_logits(logits, labels, frames_lengths, labels_lengths, average_frames=False, reduction="none",
                          blank=0, fastemit_lambda=0.0, compact=False, rnnt_type="regular", delay_penalty=0.0,
                          use_hat_loss=False):
    """``rnnt_loss(log_softmax(logits, -1), ...)`` in three dense passes instead of seven; the gradient is w.r.t. the
    LOGITS.  Dense (N,T,U,V) layout, float32 or bfloat16 (what ``torch.autocast(dtype=torch.bfloat16)`` makes of the
    joint network's output); other arguments as in ``rnnt_loss``.  Agrees with ``torch.log_softmax`` + the reference
    to 1e-5 (costs, relative) / 1e-4 (gradients), not bit for bit.

    bfloat16 logits: costs and the loss are float32, ``logits.grad`` is bfloat16, all arithmetic is float32.  The costs
    equal those of float32 logits with the same values bit for bit, and the gradient is their float32 gradient rounded
    to bfloat16 once (logits at 8-byte aligned addresses, as torch allocates them; include/rnnt_b200.h).

    ``compact=True``: ``logits`` is (STU, V), float32 or bfloat16, rows in ``joint_pack``'s order
    (STU = sum frames_lengths * (labels_lengths + 1)); ``labels`` is (sum labels_lengths,) int32, as for
    ``rnnt_loss(compact=True)``, and so are the shape checks and ``compact_hints``.  Costs are float32, the gradient is
    w.r.t. the packed logits and has their dtype.

    ``rnnt_type`` and ``delay_penalty`` are k2's (``rnnt_loss(..., rnnt_type=, delay_penalty=)``), dense layout only:
      - ``"regular"`` (default): the lattice above, a label edge stays in its frame.
      - ``"modified"``: one symbol per frame, a label edge (t,u)->(t+1,u+1) also leaves the frame; a lattice with more
        labels than frames has no path (cost +inf).
      - ``"constrained"``: modified, with each label edge weighted by its log-prob plus the blank log-prob of the cell it
        reaches in the same frame (k2's ``px += py[:, 1:, :]``).
      - ``delay_penalty`` (lambda >= 0): adds lambda * ((T_n - 1) / 2 - t) to every label log-prob of frame t, so that
        paths emitting earlier score higher (icefall's streaming recipes).  The costs include the penalty, as k2's do.
    Non-regular types take no FastEmit (k2 has none); regular + penalty + FastEmit compose.  A lattice with invalid
    lengths gets cost NaN, one without a finite path +inf, one with a NaN in its live log-probs NaN, with zero, zero and
    NaN gradients; the one-symbol-per-frame types take label dimensions up to 25599 (include/rnnt_b200.h).  Bad values
    raise ValueError before any launch.  ``rnnt_align_from_logits`` gives the best path on the same lattice.

    ``use_hat_loss=True`` (k2's name): the Hybrid Autoregressive Transducer's normalisation (HAT; Variani et al. 2020,
    arXiv:2003.07705) in place of log_softmax, as k2's ``get_hat_logprobs`` (and NeMo's ``HATJoint``) factorise the
    joint: P(blank) = sigmoid(x[blank]) and P(y | not blank) a softmax over the non-blank logits.  In float32 per row
    x, with lse_nb the normaliser over the columns v != blank (summed as a row whose blank logit is -inf, so every
    non-blank logit -inf gives NaN), s = log1p(exp(-|x[blank]|)):
      - blank log-prob b = min(x[blank], 0) - s = logsigmoid(x[blank]);
      - label log-prob l = (x[y] - lse_nb) + (min(-x[blank], 0) - s) = log_softmax_nb(x)[y] + logsigmoid(-x[blank]).
    Everything downstream of (b, l) is unchanged: ``rnnt_type``, ``delay_penalty``, FastEmit, the classes, the compact
    layout and the hints.  The gradient applies the HAT Jacobian to the (blank, label) gradients (gb, gl):
    gl * ([v == y] - exp(x[v] - lse_nb)) at a non-blank column, gb * sigmoid(-x[blank]) - gl * sigmoid(x[blank]) at
    the blank column (plus gl where the label is the blank); a row without gradient gets zeros, NaN at the non-blank
    columns where lse_nb is NaN and at the blank column where x[blank] is NaN, as autograd of the composition gives.
    One difference from log_softmax follows: a NaN confined to the non-blank columns of a last-column row (u = U_n - 1)
    reaches only l, which no lattice reads there, so the cost stays finite.  Needs V >= 2 (else ValueError); a
    ``use_hat_loss`` that is not a bool is a ValueError.  The implementation follows k2's ``get_hat_logprobs``; it was
    not tested against k2 or NeMo."""
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert isinstance(blank, int)
    assert isinstance(compact, bool)
    assert not labels.requires_grad and not frames_lengths.requires_grad and not labels_lengths.requires_grad
    kind, lam = _path_type("rnnt_loss_from_logits", rnnt_type, delay_penalty, fastemit_lambda, compact)
    hat = _use_hat("rnnt_loss_from_logits", use_hat_loss, logits)
    if compact:
        costs = RNNTLossFromLogitsCompact.apply(logits, labels, frames_lengths, labels_lengths, blank, fastemit_lambda,
                                                hat)
    else:
        costs = RNNTLossFromLogits.apply(logits, labels, frames_lengths, labels_lengths, blank, fastemit_lambda, kind,
                                         lam, hat)
    return _reduce(costs, frames_lengths, average_frames, reduction)


class RNNTLossPruned(torch.autograd.Function):
    """``RNNTLossFromLogits`` on the (N,T,S,V) logits of a joint evaluated in a window of S labels per frame.  Forward
    reads the window rows once and runs the recurrence on the full (N,T,U) lattice, with the edges out of the cells
    outside the windows removed; it keeps lse (N,T,S) and the (N,T,U,2) pair gradients.  Backward writes d loss /
    d logits (N,T,S,V), of the logits' dtype.  ``hat``: the HAT normalisation in place of log_softmax."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, ranges, blank=0, fastemit_lambda=0.0, rnnt_type=0,
                delay_penalty=0.0, hat=False):
        need = ctx.needs_input_grad[0]
        costs, lse, pg = _C.rnnt_logits_pruned_forward(logits, labels, frames_lengths, labels_lengths, ranges, blank,
                                                       fastemit_lambda, need, 0, rnnt_type, delay_penalty, hat)
        if need:
            ctx.save_for_backward(logits, lse, pg, labels, ranges)
            ctx.blank = blank
            ctx.hat = hat
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels, ranges = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_logits_pruned_backward(logits, lse, pg, labels, ranges, go, ctx.blank, ctx.hat)
        return g, None, None, None, None, None, None, None, None, None


def rnnt_loss_pruned(logits, labels, frames_lengths, labels_lengths, ranges, average_frames=False, reduction="none",
                     blank=0, fastemit_lambda=0.0, rnnt_type="regular", delay_penalty=0.0, use_hat_loss=False):
    """Pruned RNN-T loss: the transducer loss from a joint network evaluated only in a window of S label columns per
    frame, which takes about U/S times less memory and traffic than the full (N,T,U,V) joint output.

    Args:
        logits: (N, T, S, V) float32 or bfloat16, not normalised.
        labels: (N, U-1) int32, as for ``rnnt_loss``; U = labels.size(1) + 1 is the full lattice's width.
        frames_lengths, labels_lengths: (N,) int32.
        ranges: (N, T) int32; ranges[n, t] is the first label column of frame t's window.
        average_frames, reduction, blank, fastemit_lambda: as in ``rnnt_loss_from_logits``.
        rnnt_type, delay_penalty: k2's, as in ``rnnt_loss_from_logits``, on the full lattice with the edges out of the
            cells outside the windows removed.  A constrained label edge also reads the blank of the cell it
            reaches, so it is removed when that cell lies outside its frame's window.
        use_hat_loss: k2's flag, as in ``rnnt_loss_from_logits``: the HAT normalisation of each window row in place of
            log_softmax (lse then holds the non-blank normaliser).  A HAT pipeline takes its ``ranges`` from the
            regular ``rnnt_loss_simple``, which is unchanged.

    Row (n, t, s) of ``logits`` is lattice cell (t, u = ranges[n, t] + s) when t < frames_lengths[n] and
    0 <= u <= labels_lengths[n]; any other row is padding.  Frame t's window is {u : r <= u < r + S} clipped to the
    lattice; windows need not be monotone or connected, and r < 0 or r + S > labels_lengths[n] + 1 simply clip.  The
    loss is the RNN-T loss of lattice n in which the blank edge (t,u)->(t+1,u) and the label edge (t,u)->(t,u+1) of an
    in-window cell carry log_softmax(logits[n,t,s]) at ``blank`` and at labels[n,u], and every edge out of a cell outside
    its frame's window is removed.  This is k2's ``rnnt_loss_pruned(..., rnnt_type="regular")`` with k2's
    ``ranges[:, :, 0]`` as ``ranges``.  ``rnnt_loss_simple(..., prune_range=S)`` returns such ranges, chosen from the
    occupation probabilities of the simple (factorised) joint, as k2's ``get_rnnt_prune_ranges`` does.

    Costs are float32; the gradient is w.r.t. ``logits``, of their dtype (bfloat16: the float32 gradient of the
    widened logits rounded once).  Padding rows get exact zeros, or NaN where the row's normaliser is NaN.  A lattice
    with no path left gets, with ``rnnt_type="regular"``, the dense classes of ``rnnt_loss_from_logits``: cost NaN
    (+inf when it has one frame or no labels); with "modified" or "constrained", cost +inf and exactly zero gradient
    rows, as for more labels than frames.  No host synchronisation: the step can be captured in a CUDA graph."""
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert isinstance(blank, int)
    assert not labels.requires_grad and not frames_lengths.requires_grad and not labels_lengths.requires_grad
    assert not ranges.requires_grad
    kind, lam = _path_type("rnnt_loss_pruned", rnnt_type, delay_penalty, fastemit_lambda)
    hat = _use_hat("rnnt_loss_pruned", use_hat_loss, logits)
    costs = RNNTLossPruned.apply(logits, labels, frames_lengths, labels_lengths, ranges, blank, fastemit_lambda, kind,
                                 lam, hat)
    return _reduce(costs, frames_lengths, average_frames, reduction)


class RNNTLossTDT(torch.autograd.Function):
    """The Token-and-Duration Transducer loss from (N,T,U,V+D) joint logits.  Forward reads the logits once (two
    normalisers per cell, the 2 + D log-probs the recurrence needs), runs alpha and beta on the lattice and keeps lse
    (N,T,U,2) and the per-cell posteriors (N,T,U,2+D); backward reads the logits again and writes d loss / d logits, of
    their dtype."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, durations, sigma=0.0, blank=0):
        need = ctx.needs_input_grad[0]
        costs, lse, pg = _C.rnnt_tdt_forward(logits, labels, frames_lengths, labels_lengths, list(durations), sigma,
                                             blank, need)
        if need:
            ctx.save_for_backward(logits, lse, pg, labels)
            ctx.durations = list(durations)
            ctx.blank = blank
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_tdt_backward(logits, lse, pg, labels, ctx.durations, go, ctx.blank)
        return g, None, None, None, None, None, None


class RNNTLossTDTCompact(torch.autograd.Function):
    """``RNNTLossTDT`` on compact (STU,V+D) logits in ``joint_pack``'s row order: a packed TDT joint feeds the loss
    without padding.  Forward keeps lse (STU,2), the posteriors (STU,2+D) and the compact prefix sums (16 bytes per
    lattice); backward writes d loss / d logits, of the logits' dtype.  Inside ``compact_hints`` the forward has no host
    sync (CUDA-graph capturable)."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, durations, sigma=0.0, blank=0):
        need = ctx.needs_input_grad[0]
        hints = _hints()
        costs, lse, pg, prefix = _C.rnnt_tdt_compact_forward(logits, labels, frames_lengths, labels_lengths,
                                                             list(durations), sigma, blank, need, hints[0], hints[1])
        if need:
            ctx.save_for_backward(logits, lse, pg, labels, frames_lengths, labels_lengths, prefix)
            ctx.durations = list(durations)
            ctx.blank = blank
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels, xn, yn, prefix = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_tdt_compact_backward(logits, lse, pg, labels, xn, yn, prefix, ctx.durations, go, ctx.blank)
        return g, None, None, None, None, None, None


def _tdt_args(fn, logits, durations, sigma, blank, compact):
    """The argument checks of ``rnnt_loss_tdt`` and ``rnnt_align_tdt`` (``fn`` names the caller in the messages):
    durations, sigma, the logits' shape and blank.  Returns the durations as a tuple."""
    if not isinstance(durations, (list, tuple)) or not durations or \
            any(isinstance(d, bool) or not isinstance(d, int) for d in durations):
        raise ValueError("%s: durations must be a non-empty list or tuple of ints, got %r" % (fn, durations))
    if any(d < 0 or d > 16 for d in durations) or any(b <= a for a, b in zip(durations, durations[1:])) \
            or max(durations) == 0:
        raise ValueError("%s: durations must be strictly increasing, in [0, 16], with at least one > 0, "
                         "got %r" % (fn, durations))
    if isinstance(sigma, bool) or not isinstance(sigma, (int, float)) or not math.isfinite(sigma) or sigma < 0:
        raise ValueError("%s: sigma must be a finite number >= 0, got %r" % (fn, sigma))
    assert isinstance(compact, bool)
    if logits.dim() != (2 if compact else 4) or logits.size(-1) <= len(durations):
        raise ValueError("%s: logits must be %s with V >= 1, D = len(durations) = %d, got shape %s"
                         % (fn, "(STU, V + D)" if compact else "(N, T, U, V + D)", len(durations),
                            tuple(logits.shape)))
    if isinstance(blank, bool) or not isinstance(blank, int) or not 0 <= blank < logits.size(-1) - len(durations):
        raise ValueError("%s: blank must be an int in [0, V), got %r" % (fn, blank))
    return tuple(durations)


def rnnt_loss_tdt(logits, labels, frames_lengths, labels_lengths, durations, sigma=0.0, average_frames=False,
                  reduction="none", blank=0, compact=False):
    """Token-and-Duration Transducer loss (TDT, Xu et al. 2023, arXiv:2304.06795), the loss of NeMo's Parakeet-TDT
    models, from the joint network's logits.  Follows NeMo's definition (``TDTLossPytorch``: the same alpha recursion
    and terminal sum); not tested against NeMo.

    Args:
        logits: (N, T, U, V + D) float32 or bfloat16, NeMo's layout: V token logits (blank included), then D duration
            logits, D = len(durations).  U = labels.size(1) + 1.  ``compact=True``: (STU, V + D), see below.
        labels: (N, U-1) int32; frames_lengths, labels_lengths: (N,) int32, as for ``rnnt_loss_from_logits``.
        durations: list or tuple of ints, strictly increasing, in [0, 16], at least one > 0 (else ValueError), e.g.
            [0, 1, 2, 3, 4].  Host values: they reach the kernels as launch parameters.
        sigma: NeMo's logit under-normalisation, a finite float >= 0 (else ValueError).
        average_frames, reduction: as in ``rnnt_loss_from_logits``.
        blank: in [0, V).
        compact: the ragged layout of ``rnnt_loss_from_logits(compact=True)``.

    Lattice n has Tn = frames_lengths[n] frames and Un = labels_lengths[n] + 1 columns.  Cell (t, u) has
    lt = log_softmax(logits[n,t,u,:V]) - sigma, the token log-probs, and ld = log_softmax(logits[n,t,u,V:]), the
    duration log-probs.  Edges out of cell (t, u), with t < Tn and u < Un:

    * blank edge, for each j with d = durations[j] > 0, weight lt[blank] + ld[j]: to (t + d, u) if t + d < Tn; terminal
      if u = Un - 1 and t + d = Tn; otherwise no edge.
    * label edge, for u < Un - 1 and each j (d = 0 included), weight lt[labels[n,u]] + ld[j]: to (t + d, u + 1) if
      t + d < Tn; otherwise no edge.  A path therefore always ends with a blank.

    P is the sum, over paths from (0, 0) to a terminal edge, of exp(sum of edge weights); cost[n] = -log P.  Edge
    posterior gamma_e = exp(alpha(src) + w_e + beta(dst) - log P), with beta = 0 after a terminal edge.  Per cell, Pb is
    the sum of gamma over its blank edges, Pl over its label edges, Pd[j] over its edges of duration durations[j], and
    occ = Pb + Pl = sum Pd.  The gradient of the cost w.r.t. the logits, times grad_output[n] (and the reduction's
    weights), is occ * softmax_tok[v] - Pb [v = blank] - Pl [v = label] on the tokens and occ * softmax_dur[j] - Pd[j]
    on the durations; a label equal to blank gets both terms, as autograd gives.

    Degenerate input, without host synchronisation:

    * padding rows (t >= Tn or u >= Un) are never read, so a NaN there changes nothing; their gradient is exactly 0;
    * invalid lengths (Tn outside [1, T] or labels_lengths[n] outside [0, U-1]) or a live label outside [0, V): cost
      NaN, all-zero gradient rows;
    * no path of finite log-probability, structurally (e.g. Tn < min(d > 0)) or through -inf token or duration logits:
      cost +inf, all-zero gradient rows;
    * a NaN or +inf in a live row, or a live row whose token or duration logits are all -inf: cost NaN and NaN gradients
      on that lattice's live rows; every other lattice of the batch is bit-identical to a batch without it.

    Costs are float32; ``logits.grad`` has the logits' dtype.  bfloat16: costs equal those of the float32 logits with
    the same values bit for bit, and the gradient is their float32 gradient rounded once.  Deterministic (no atomics),
    no host synchronisation: a step can be captured in a CUDA graph.  ``set_lse_mode`` does not apply.

    ``compact=True``: ``logits`` is (STU, V + D), float32 or bfloat16, rows in ``joint_pack``'s order (row (n, t, u) at
    sum_{m<n} Tm * Um + t * Un + u, STU = sum frames_lengths * (labels_lengths + 1)), and ``labels`` is
    (sum labels_lengths,) int32, concatenated in lattice order.  Semantics, degenerate classes and gradient are those of
    the dense call: costs, the normalisers, the posteriors and the gradient are bit for bit those of the same rows placed
    in a padded tensor at the same element offset modulo 4.  Without ``compact_hints`` the call makes one small
    device->host copy to check STU and ``labels.numel()`` against the lengths; inside ``compact_hints(max_T, max_U)`` it
    makes none (forward and backward can be captured in a CUDA graph), and a sample exceeding the hints, or one whose
    rows would run past STU, gets cost NaN and zero gradient rows.  Rows of no valid lattice get exact zeros.  A packed
    TDT joint::

        x = joint_pack(f, g, frames_lengths, labels_lengths)          # (STU, H), no padding
        logits = joint(x)                                             # (STU, V + D)
        loss = rnnt_loss_tdt(logits, labels_c, frames_lengths, labels_lengths, [0, 1, 2, 3, 4], compact=True,
                             reduction="mean")

    Not offered: ``fastemit_lambda`` and NeMo's ``omega`` mixing with the regular transducer loss.  The multi-blank
    transducer loss is ``rnnt_loss_multiblank``.  The best path itself (token frames and durations) is
    ``rnnt_align_tdt``."""
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert not labels.requires_grad and not frames_lengths.requires_grad and not labels_lengths.requires_grad
    durations = _tdt_args("rnnt_loss_tdt", logits, durations, sigma, blank, compact)
    fn = RNNTLossTDTCompact if compact else RNNTLossTDT
    costs = fn.apply(logits, labels, frames_lengths, labels_lengths, durations, float(sigma), blank)
    return _reduce(costs, frames_lengths, average_frames, reduction)


class RNNTLossMultiblank(torch.autograd.Function):
    """The multi-blank transducer loss from (N,T,U,V) joint logits.  Forward reads the logits once (one normaliser per
    cell, the 2 + B log-probs the recurrence needs), runs alpha and beta on the lattice and keeps lse (N,T,U) and the
    per-cell edge posteriors (N,T,U,2+B); backward reads the logits again and writes d loss / d logits, of their
    dtype."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, big_blank_durations, sigma, blank):
        need = ctx.needs_input_grad[0]
        costs, lse, pg = _C.rnnt_multiblank_forward(logits, labels, frames_lengths, labels_lengths,
                                                    list(big_blank_durations), sigma, blank, need)
        if need:
            ctx.save_for_backward(logits, lse, pg, labels)
            ctx.durations = list(big_blank_durations)
            ctx.blank = blank
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_multiblank_backward(logits, lse, pg, labels, ctx.durations, go, ctx.blank)
        return g, None, None, None, None, None, None


class RNNTLossMultiblankCompact(torch.autograd.Function):
    """``RNNTLossMultiblank`` on compact (STU,V) logits in ``joint_pack``'s row order.  Forward keeps lse (STU), the
    posteriors (STU,2+B) and the compact prefix sums (16 bytes per lattice).  Inside ``compact_hints`` the forward has
    no host sync (CUDA-graph capturable)."""

    @staticmethod
    def forward(ctx, logits, labels, frames_lengths, labels_lengths, big_blank_durations, sigma, blank):
        need = ctx.needs_input_grad[0]
        hints = _hints()
        costs, lse, pg, prefix = _C.rnnt_multiblank_compact_forward(logits, labels, frames_lengths, labels_lengths,
                                                                    list(big_blank_durations), sigma, blank, need,
                                                                    hints[0], hints[1])
        if need:
            ctx.save_for_backward(logits, lse, pg, labels, frames_lengths, labels_lengths, prefix)
            ctx.durations = list(big_blank_durations)
            ctx.blank = blank
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        logits, lse, pg, labels, xn, yn, prefix = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        g = _C.rnnt_multiblank_compact_backward(logits, lse, pg, labels, xn, yn, prefix, ctx.durations, go, ctx.blank)
        return g, None, None, None, None, None, None


def _multiblank_args(fn, logits, big_blank_durations, sigma, blank, compact):
    """The argument checks of ``rnnt_loss_multiblank`` and ``rnnt_align_multiblank`` (``fn`` names the caller in the
    messages): the durations, sigma, the logits' shape and blank.  Returns
    (durations as a tuple, the standard blank's column)."""
    d = big_blank_durations
    if not isinstance(d, (list, tuple)) or not d or any(isinstance(x, bool) or not isinstance(x, int) for x in d):
        raise ValueError("%s: big_blank_durations must be a non-empty list or tuple of ints, got %r" % (fn, d))
    if any(x < 2 or x > 16 for x in d) or any(b <= a for a, b in zip(d, d[1:])):
        raise ValueError("%s: big_blank_durations must be strictly increasing, each in [2, 16], got %r" % (fn, d))
    if isinstance(sigma, bool) or not isinstance(sigma, (int, float)) or not math.isfinite(sigma) or sigma < 0:
        raise ValueError("%s: sigma must be a finite number >= 0, got %r" % (fn, sigma))
    assert isinstance(compact, bool)
    if logits.dim() != (2 if compact else 4) or logits.size(-1) <= len(d):
        raise ValueError("%s: logits must be %s with V > B = len(big_blank_durations) = %d, got shape %s"
                         % (fn, "(STU, V)" if compact else "(N, T, U, V)", len(d), tuple(logits.shape)))
    V = logits.size(-1)
    if blank is None:
        blank = V - 1
    if isinstance(blank, bool) or not isinstance(blank, int) or not len(d) <= blank < V:
        raise ValueError("%s: blank must be None or an int in [B, V) = [%d, %d), got %r" % (fn, len(d), V, blank))
    return tuple(d), blank


def rnnt_loss_multiblank(logits, labels, frames_lengths, labels_lengths, big_blank_durations, sigma=0.0,
                         average_frames=False, reduction="none", blank=None, compact=False):
    """Multi-blank transducer loss (Xu et al. 2022, "Multi-blank Transducers for Speech Recognition",
    arXiv:2211.03541), the loss of NeMo's multi-blank Conformer-Transducer, from the joint network's logits.  Follows
    NeMo's definition (``MultiblankRNNTLossPytorch``: the same alpha recursion, terminal sum, column layout and sigma);
    not tested against NeMo.

    Args:
        logits: (N, T, U, V) float32 or bfloat16.  V is the whole row: the tokens, the big blanks and the standard
            blank.  U = labels.size(1) + 1.  ``compact=True``: (STU, V), see below.
        labels: (N, U-1) int32; frames_lengths, labels_lengths: (N,) int32, as for ``rnnt_loss_from_logits``.
        big_blank_durations: list or tuple of B >= 1 ints, strictly increasing, each in [2, 16] (else ValueError),
            e.g. [2, 4, 8].  Host values: they reach the kernels as launch parameters.
        sigma: NeMo's logit under-normalisation, a finite float >= 0 (else ValueError).
        average_frames, reduction: as in ``rnnt_loss_from_logits``.
        blank: the standard blank's column; None (default) means V - 1, NeMo's layout.  Big blank i sits in column
            blank - 1 - i.  An explicit blank must lie in [B, V).
        compact: the ragged layout of ``rnnt_loss_from_logits(compact=True)``.

    Lattice n has Tn = frames_lengths[n] frames and Un = labels_lengths[n] + 1 columns.  Every edge weight is
    lp = log_softmax(logits[n,t,u,:]) - sigma at the edge's column.  Edges out of cell (t, u), with t < Tn and u < Un:

    * standard blank, weight lp[blank]: to (t + 1, u) if t + 1 < Tn; terminal if u = Un - 1 and t + 1 = Tn;
    * big blank i, d = big_blank_durations[i], weight lp[blank - 1 - i]: to (t + d, u) if t + d < Tn; terminal if
      u = Un - 1 and t + d = Tn; otherwise no edge;
    * label, for u < Un - 1, weight lp[labels[n,u]]: to (t, u + 1).

    P is the sum, over paths from (0, 0) to a terminal edge, of exp(sum of edge weights); cost[n] = -log P.  Per cell,
    the edge posteriors are P_std, P_big[i] and Pl, and occ is their sum.  The gradient of the cost w.r.t. the logits,
    times grad_output[n] (and the reduction's weights), is
    occ * softmax[v] - P_std [v = blank] - sum_i P_big[i] [v = blank - 1 - i] - Pl [v = label]; a label equal to a
    blank column gets both terms, as autograd gives.

    Degenerate input, without host synchronisation: padding rows are never read and get exact zeros; invalid lengths or
    a live label outside [0, V) give cost NaN and zero gradient rows; a NaN or +inf in a live row, or a live row that is
    all -inf, gives cost NaN and NaN on that lattice's live rows (every other lattice is bit-identical to a batch
    without it); no path of finite log-probability (only through -inf logits, as the standard blank always gives a
    path) gives cost +inf and zero gradient rows.

    Costs are float32; ``logits.grad`` has the logits' dtype.  bfloat16: costs equal those of the float32 logits with
    the same values bit for bit, and the gradient is their float32 gradient rounded once.  Deterministic (no atomics),
    no host synchronisation: a step can be captured in a CUDA graph.  ``set_lse_mode`` does not apply.

    ``compact=True``: ``logits`` is (STU, V), rows in ``joint_pack``'s order, and ``labels`` is (sum labels_lengths,)
    int32, as for ``rnnt_loss_tdt(compact=True)``, with the same ``compact_hints`` behaviour and classes: costs, the
    posteriors and the gradient are bit for bit those of the same rows placed in a padded tensor at the same element
    offset modulo 4.

    Not offered: ``fastemit_lambda``, ``rnnt_type``, ``delay_penalty`` and TDT's ``omega``.  The best path itself
    (token frames and blank counts) is ``rnnt_align_multiblank``."""
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert not labels.requires_grad and not frames_lengths.requires_grad and not labels_lengths.requires_grad
    durations, blank = _multiblank_args("rnnt_loss_multiblank", logits, big_blank_durations, sigma, blank, compact)
    fn = RNNTLossMultiblankCompact if compact else RNNTLossMultiblank
    costs = fn.apply(logits, labels, frames_lengths, labels_lengths, durations, float(sigma), blank)
    return _reduce(costs, frames_lengths, average_frames, reduction)


class RNNTLossSimple(torch.autograd.Function):
    """The simple loss of the pruned recipe: the transducer loss of the joint ``am[n,t] + lm[n,u]``, whose normaliser is
    a (T,V) x (V,U) product per lattice, so no (N,T,U,V) tensor is formed.  Forward keeps the normaliser (N,T,U), the
    row offsets of ``am`` and ``lm`` and the (N,T,U,2) pair gradients; backward writes d loss / d ``am`` and d ``lm``.
    With ``prune_range`` > 0 the forward also returns the (N,T) prune ranges (else an empty int tensor).
    ``lm_only_scale`` / ``am_only_scale``: k2's smoothing (``rnnt_loss_simple``); with either > 0 the forward also keeps
    the LM-only and AM-only normalisers and the log of the batch unigram."""

    @staticmethod
    def forward(ctx, am, lm, labels, frames_lengths, labels_lengths, blank=0, prune_range=0, lm_only_scale=0.0,
                am_only_scale=0.0, rnnt_type=0, delay_penalty=0.0):
        need = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        costs, saved, pg, ranges = _C.rnnt_simple_forward(am, lm, labels, frames_lengths, labels_lengths, blank, need,
                                                          prune_range, 0, lm_only_scale, am_only_scale, rnnt_type,
                                                          delay_penalty)
        if need:
            ctx.save_for_backward(am, lm, labels, frames_lengths, labels_lengths, saved, pg)
            ctx.blank = blank
            ctx.scales = (lm_only_scale, am_only_scale)
        ctx.mark_non_differentiable(ranges)
        return costs, ranges

    @staticmethod
    def backward(ctx, grads_output, _grad_ranges):
        am, lm, labels, xn, yn, saved, pg = ctx.saved_tensors
        go = grads_output.contiguous().to(torch.float32)
        dam, dlm = _C.rnnt_simple_backward(am, lm, labels, xn, yn, saved, pg, go, ctx.blank, *ctx.scales)
        return (dam if ctx.needs_input_grad[0] else None), (dlm if ctx.needs_input_grad[1] else None), \
            None, None, None, None, None, None, None, None, None


def _smoothing_scale(name, x):
    if isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x) or x < 0:
        raise ValueError("rnnt_loss_simple: %s must be a finite number >= 0, got %r" % (name, x))
    return float(x)


def rnnt_loss_simple(am, lm, labels, frames_lengths, labels_lengths, average_frames=False, reduction="none", blank=0,
                     prune_range=None, lm_only_scale=0.0, am_only_scale=0.0, rnnt_type="regular", delay_penalty=0.0):
    """Simple transducer loss of the pruned recipe, and the windows ``rnnt_loss_pruned`` takes.  Follows k2's
    ``rnnt_loss_simple`` + ``get_rnnt_prune_ranges`` (regular lattice), and with ``lm_only_scale`` /
    ``am_only_scale`` k2's ``rnnt_loss_smoothed``; not tested against k2.

    Args:
        am: (N, T, V) float32, the encoder output projected to the vocabulary.
        lm: (N, U, V) float32, the predictor output projected to the vocabulary; U = labels.size(1) + 1.
        labels: (N, U-1) int32; frames_lengths, labels_lengths: (N,) int32, as for ``rnnt_loss``.
        average_frames, reduction, blank: as in ``rnnt_loss_from_logits``.
        prune_range: None, or an int S >= 2: also return the (N, T) int32 ``ranges`` for
            ``rnnt_loss_pruned(..., ranges)`` with windows of S labels.
        lm_only_scale, am_only_scale: k2's smoothing scales sl, sa: finite, >= 0, sl + sa < 1 (else ValueError).
            Both 0 (the default) is the plain simple loss, with the same kernels and the same bits.
        rnnt_type, delay_penalty: k2's, as in ``rnnt_loss_from_logits`` (the penalty goes on the smoothed pairs).
            With "modified" / "constrained", ``prune_range`` may be 1 and the windows move by at most one column a frame
            (k2's ``_adjust_pruning_lower_bound(s_begin, 2)``); they are scored from the raw edge occupations, for
            "constrained" the blank edges' before their label-edge share is folded in.  The last frame's window then
            holds the last label whenever labels_lengths - prune_range + 1 <= frames_lengths - 1.

    The loss is the RNN-T loss of lattice n in which cell (t, u) has the log-probs log_softmax(am[n,t] + lm[n,u]) at
    ``blank`` and at labels[n,u].  Its normaliser is log(sum_v exp(am[n,t,v]) exp(lm[n,u,v])), a fp32 contraction over
    V (include/rnnt_b200.h gives the exact operation order); a cell whose products all underflow is clamped to
    log(FLT_MIN) plus the row maxima instead of going to -inf.  The gradient flows to ``am`` and ``lm``, deterministic.

    Smoothing (k2's ``rnnt_loss_smoothed(..., lm_only_scale=sl, am_only_scale=sa)``): with c = 1 - sl - sa, each of the
    two log-probs of cell (t, u), for k = blank or labels[n,u], becomes
    ``c * simple_k + sl * log_softmax(lm[n,u])[k] + sa * log(exp(am[n,t,k]) uni[k] / sum_v exp(am[n,t,v]) uni[v])``,
    where ``uni`` is the unigram of the batch: the mean over every row of ``lm`` (padding rows included, as in k2) of
    softmax(lm[n,u]), plus FLT_MIN.  A term whose scale is 0 is left out; k2 multiplies it by 1e-20 instead, which
    differs only where that term is +-inf or NaN.  With ``am_only_scale`` > 0 the unigram couples the batch: a NaN
    anywhere in ``lm`` makes every cost NaN, every row of ``lm`` gets a gradient, and a call on a micro-batch or a shard
    uses that part's own unigram, as k2 does with a smaller batch.  The ranges come from the smoothed lattice, as k2's
    recipes take them.  k2's own defaults are ``lm_only_scale=0.1, am_only_scale=0.1``, and icefall's recipes pass
    ``lm_only_scale=0.25, am_only_scale=0.0``: a port passes the scales explicitly.

    The ranges come from the occupation probabilities of this loss's lattice: each frame takes the window of S columns
    with the most occupation, then the windows are made to start at 0, never move back, move by at most S-1 columns a
    frame and end on the last label.  The call returns ``(loss, ranges)`` then.  The ranges carry no gradient.

    bfloat16 ``am`` / ``lm`` are refused: these tensors are small beside the joint, and the loss is run in float32.
    Lengths outside (1..T, 0..U-1) give cost NaN, zero gradient rows and ranges 0 (with ``am_only_scale`` > 0 their
    ``lm`` rows still get the unigram's gradient).  No host synchronisation: the step can be captured in a CUDA graph.

    Typical use, with no (N, T, U, V) tensor anywhere::

        simple, ranges = rnnt_loss_simple(am, lm, labels, xn, yn, reduction="sum", prune_range=5,
                                          lm_only_scale=0.25, am_only_scale=0.0)
        idx = (ranges[:, :, None] + torch.arange(5, device=ranges.device)).clamp(max=lm_in.size(1) - 1)
        lm_win = lm_in[torch.arange(N, device=lm_in.device)[:, None, None], idx]     # (N, T, 5, H)
        logits = joint(enc_in[:, :, None] + lm_win)                                  # (N, T, 5, V)
        loss = simple_scale * simple + rnnt_loss_pruned(logits, labels, xn, yn, ranges, reduction="sum")
    """
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert isinstance(blank, int)
    assert not labels.requires_grad and not frames_lengths.requires_grad and not labels_lengths.requires_grad
    if am.dtype != torch.float32 or lm.dtype != torch.float32:
        raise TypeError("rnnt_loss_simple: am and lm must be float32, got %s and %s (bfloat16 is not supported; "
                        "run this loss outside autocast or cast with .float())" % (am.dtype, lm.dtype))
    kind, lam = _path_type("rnnt_loss_simple", rnnt_type, delay_penalty)
    least = 2 if kind == 0 else 1
    if prune_range is not None and (isinstance(prune_range, bool) or not isinstance(prune_range, int)
                                    or prune_range < least):
        raise ValueError("rnnt_loss_simple: prune_range must be None or an int >= %d, got %r" % (least, prune_range))
    sl = _smoothing_scale("lm_only_scale", lm_only_scale)
    sa = _smoothing_scale("am_only_scale", am_only_scale)
    # the kernels take the scales as float32: the check is on the values they see
    if torch.tensor(sl, dtype=torch.float32).item() + torch.tensor(sa, dtype=torch.float32).item() >= 1.0:
        raise ValueError("rnnt_loss_simple: lm_only_scale + am_only_scale must be < 1, got %r + %r" % (sl, sa))
    costs, ranges = RNNTLossSimple.apply(am, lm, labels, frames_lengths, labels_lengths, blank, prune_range or 0, sl, sa,
                                         kind, lam)
    costs = _reduce(costs, frames_lengths, average_frames, reduction)
    return costs if prune_range is None else (costs, ranges)


class JointPack(torch.autograd.Function):
    """x[(n,t,u), :] = f[n,t,:] + g[n,u,:] in the compact (ragged) row order that ``rnnt_loss(compact=True)`` takes --
    the joint network's input without padding (the reference's benchmark2.py:37-50 builds it with a python loop over
    the batch).  One kernel forward, two deterministic reductions backward."""

    @staticmethod
    def forward(ctx, f, g, lf, lg, stu=-1):
        x, mem_pref = _C.rnnt_joint_pack(f.contiguous(), g.contiguous(), lf, lg, int(stu))
        ctx.save_for_backward(lf, lg, mem_pref)
        ctx.shape = (f.size(1), g.size(1))
        return x

    @staticmethod
    def backward(ctx, dx):
        lf, lg, mem_pref = ctx.saved_tensors
        df, dg = _C.rnnt_joint_pack_backward(dx.contiguous().float(), lf, lg, mem_pref, ctx.shape[0], ctx.shape[1])
        return df, dg, None, None, None


def joint_pack(f, g, frames_lengths, labels_lengths, stu=None):
    """f (N,T,H) encoder output, g (N,U+1,H) predictor output -> (STU,H), STU = sum frames_lengths*(labels_lengths+1):
    the packed input of the joint network whose (STU,V) log-softmax output goes to ``rnnt_loss(..., compact=True)``.
    ``stu``: pass STU when known to avoid the one device->host copy that sizes the output."""
    return JointPack.apply(f, g, frames_lengths, labels_lengths, -1 if stu is None else int(stu))


class RNNTLossEager(torch.autograd.Function):
    """Reference-shaped variant: dense gradients are produced in forward (one fused pass) and
    scaled in backward, exactly like the reference's RNNTLoss (__init__.py:11-24)."""

    @staticmethod
    def forward(ctx, log_probs, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0):
        costs, ctx.grads = _C.rnnt_loss(xs=log_probs, ys=labels, xn=frames_lengths, yn=labels_lengths,
                                        blank=blank, fastemit_lambda=fastemit_lambda)
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        grads_output = grads_output.view(-1, 1, 1, 1).to(ctx.grads)
        return ctx.grads.mul_(grads_output), None, None, None, None, None


_tls = threading.local()


def _hints():
    """(max_T, max_U) of the enclosing ``compact_hints``, or (0, 0): none."""
    return getattr(_tls, "hints", None) or (0, 0)


@contextlib.contextmanager
def compact_hints(max_T, max_U):
    """Inside this context ``rnnt_loss(compact=True)`` trusts the caller's upper bounds of ``frames_lengths`` and
    ``labels_lengths + 1`` and skips the shape validation that needs a device->host copy of the length sums (the
    reference does four ``.item()`` syncs there, binding.cpp:132-146): the forward then has no host sync at all
    and can be captured into a CUDA graph.  A sample exceeding the bounds gets cost NaN."""
    prev = getattr(_tls, "hints", None)
    _tls.hints = (int(max_T), int(max_U))
    try:
        yield
    finally:
        _tls.hints = prev


class RNNTLossCompact(torch.autograd.Function):
    """Compact (ragged) layout.  Reference: ``RNNTLossCompact`` (__init__.py:26-54)."""

    @staticmethod
    def forward(ctx, log_probs, labels, frames_lengths, labels_lengths, blank=0, fastemit_lambda=0.0,
                enable_grad: bool = True):
        hints = _hints()
        costs, grads, loc = _C.rnnt_loss_compact(
            xs=log_probs, ys=labels, xn=frames_lengths, yn=labels_lengths, blank=blank,
            fastemit_lambda=fastemit_lambda, required_grad=enable_grad, max_T=hints[0], max_U=hints[1])
        if enable_grad:
            cumlen = torch.cumsum(frames_lengths * (labels_lengths + 1), dim=0, dtype=torch.int32)
            ctx.V = log_probs.size(-1)
            ctx.blank = blank
            ctx.save_for_backward(grads, loc, cumlen)
        return costs

    @staticmethod
    def backward(ctx, grads_output):
        grads, loc, cumlen = ctx.saved_tensors
        grads_input = _C.rnnt_loss_compact_backward(grads_output.contiguous().float(), grads, cumlen, loc,
                                                    ctx.V, ctx.blank)
        return grads_input, None, None, None, None, None, None


def rnnt_loss(log_probs, labels, frames_lengths, labels_lengths, average_frames=False, reduction="none",
              blank=0, gather=False, fastemit_lambda=0.0, compact=False):
    """The RNN-Transducer loss (same signature and semantics as the reference, __init__.py:57-143).

    Args:
        log_probs: (N, T, U, V) float32 log-softmaxed joint output; compact: (STU, V).  The dense path
            (gather=False, compact=False) also takes bfloat16: bf16 in, bf16 gradient out, float32 costs and
            arithmetic (the reference is float32-only, binding.cpp:17-19).
        labels: (N, U-1) int32; compact: (sum(labels_lengths),).
        frames_lengths, labels_lengths: (N,) int32.
        average_frames: divide each sample's loss by its number of frames.
        reduction: 'none' | 'mean' | 'sum' | None.
        blank: blank label id.
        gather: the reference's memory-saving mode: only a (N,T,U,2) gradient lives between forward and
            backward (the dense one is emitted by backward); follows torch.gather's backward for a label
            equal to ``blank`` (the two gradients add).  ``gather=False`` (default) is the fast path: one
            kernel launch produces loss and dense gradient.
        fastemit_lambda: FastEmit regularisation (scales label gradients by 1+lambda).
        compact: ragged layout, STU = sum(frames_lengths * (labels_lengths + 1)).
    """
    assert average_frames is None or isinstance(average_frames, bool)
    assert reduction is None or reduction in ("none", "mean", "sum")
    assert isinstance(blank, int)
    assert isinstance(gather, bool)

    assert not labels.requires_grad, "labels does not require gradients"
    assert not frames_lengths.requires_grad, "frames_lengths does not require gradients"
    assert not labels_lengths.requires_grad, "labels_lengths does not require gradients"

    if compact:
        costs = RNNTLossCompact.apply(log_probs.float(), labels, frames_lengths, labels_lengths, blank,
                                      fastemit_lambda,
                                      (log_probs.requires_grad and torch.is_grad_enabled()))
    elif gather:
        assert log_probs.dtype == torch.float32, "gather=True takes float32 log_probs (bfloat16: gather=False)"
        costs = RNNTLossGather.apply(log_probs, labels, frames_lengths, labels_lengths, blank, fastemit_lambda)
    else:
        # dense path: the reduction below is folded into the one kernel launch (see RNNTLoss)
        if reduction not in ("none", "mean", "sum", None):
            raise ValueError(
                f"Unknown reduction method: {reduction}, expected to be one of ['mean', 'sum', 'none']")
        reduce = reduction in ("mean", "sum")
        weights = None                                   # float32 also for bfloat16 log_probs (costs are float32)
        if average_frames:
            weights = 1.0 / frames_lengths.to(torch.float32)
        if reduction == "mean":
            n = max(int(log_probs.size(0)), 1)
            weights = torch.full((log_probs.size(0),), 1.0 / n, dtype=torch.float32, device=log_probs.device) \
                if weights is None else weights / n
        return RNNTLoss.apply(log_probs, labels, frames_lengths, labels_lengths, blank, fastemit_lambda, weights,
                              reduce)

    if average_frames:
        costs = costs / frames_lengths.to(log_probs)

    if reduction == "none" or reduction is None:
        return costs
    elif reduction == "sum":
        return costs.sum()
    elif reduction == "mean":
        return costs.mean()
    else:
        raise ValueError(
            f"Unknown reduction method: {reduction}, expected to be one of ['mean', 'sum', 'none']")


def rnnt_align(log_probs, labels, frames_lengths, labels_lengths, blank=0, compact=False):
    """Viterbi forced alignment: the single best alignment of the labels to the frames on the RNN-T lattice, for token
    timestamps, emission latency (what ``fastemit_lambda`` tunes), alignment-restricted targets or data debugging.

    Inputs are those of ``rnnt_loss``: dense (N, T, U, V) log-probs, float32 or bfloat16, with labels (N, U-1); or
    ``compact=True``: (STU, V) log-probs, float32 or bfloat16, with labels (sum(labels_lengths),), honouring
    ``compact_hints``.  frames_lengths, labels_lengths (N,) int32.

    Returns ``(scores, frames)``:
      * ``scores`` (N,) float32: the largest path score.  A path starts at (0, 0), adds blank[t, u] for each step
        (t, u) -> (t+1, u) and label[t, u] for each step (t, u) -> (t, u+1), and ends with blank[Tn-1, Un-1]; its
        score is the float32 sum of those log-probs added left to right in path order.
      * ``frames`` int32, dense (N, U-1), compact (sum(labels_lengths),) in the labels' order: frames[n, u] is the
        frame t at which the best path emits label u (its edge (t, u) -> (t, u+1)); non-decreasing, in [0, Tn-1], and
        -1 for u >= labels_lengths[n].

    Choosing between the two predecessors of a cell, the label edge wins iff its candidate is larger or the blank
    candidate is NaN: a NaN candidate loses to any number, and on an exact tie the blank edge wins, so each label is
    emitted as early as the ties allow.  A lattice with no path above -inf gets score -inf, one whose every path is NaN
    gets NaN; lengths outside (1..T, 1..U-1 labels; compact: outside ``compact_hints``) get score NaN.  All of these
    get frames -1.  No autograd.  No host synchronisation in the dense layout and, inside ``compact_hints``, in the
    compact one (CUDA-graph capturable); without hints the compact call makes one 16-byte device->host copy.

    From joint logits, ``rnnt_align_from_logits`` gives the same result without a dense ``log_softmax`` tensor, and
    also on k2's "modified" and "constrained" lattices and with ``delay_penalty``."""
    assert isinstance(blank, int)
    assert isinstance(compact, bool)
    if compact:
        hints = _hints()
        return _C.rnnt_align_compact(log_probs, labels, frames_lengths, labels_lengths, blank, hints[0], hints[1])
    return _C.rnnt_align_dense(log_probs, labels, frames_lengths, labels_lengths, blank)


def rnnt_align_from_logits(logits, labels, frames_lengths, labels_lengths, blank=0, compact=False,
                           rnnt_type="regular", delay_penalty=0.0, use_hat_loss=False):
    """Viterbi forced alignment straight from joint logits, on the lattice of ``rnnt_loss_from_logits`` with the same
    ``rnnt_type`` and ``delay_penalty``: the single best path of each lattice and the frame of each label, without the
    dense ``log_softmax`` tensor that ``rnnt_align`` needs.  For the one-symbol-per-frame types this is the alignment
    of the lattice the model was trained on, and with a penalty it shows the emission latency the penalty tunes.

    Inputs and argument checks are those of ``rnnt_loss_from_logits``: dense (N, T, U, V) logits, float32 or bfloat16,
    with labels (N, U-1) int32; or ``compact=True``: (STU, V) rows in ``joint_pack``'s order with labels
    (sum(labels_lengths),), honouring ``compact_hints`` (``rnnt_type="regular"`` and ``delay_penalty=0`` only, as for
    the loss).  No autograd: the outputs are not differentiable and ``logits.requires_grad`` is ignored.

    Edge weights: cell (t, u) has the pair b = logit[blank] - lse and l = logit[label] - lse in float32, lse the
    normaliser of the loss's own pass, so they are bit for bit the loss's; a penalty is added to them exactly as the
    loss adds it; the constrained label weight is l(t, u) + b(t, u+1).  A path's score is the float32 left fold
    ``acc = acc + w`` over its edges; the max-plus recurrence adds in that order and so gives the largest one exactly.
      - ``"regular"``: ``rnnt_align``'s lattice, tie rule, classes and frames on these pairs, so the result equals
        ``rnnt_align(logits.float() - lse[..., None])`` bit for bit (with the penalty on the label columns).
      - ``"modified"`` / ``"constrained"``: a label edge (t, u) -> (t+1, u+1) also leaves the frame; alpha(0, 0) = 0,
        the score is alpha(Tn, Un-1), and the label edge wins iff its candidate is larger or the blank one is NaN.
        Frames are strictly increasing, in [0, Tn-1]; a lattice with more labels than frames gets score -inf.  Dense
        only, with U <= 25600.

    Returns ``(scores, frames)``: ``scores`` (N,) float32, the best path's score; ``frames`` int32, dense (N, U-1),
    compact (sum(labels_lengths),): frames[n, u] is the frame of the best path's edge for label u, -1 for
    u >= labels_lengths[n].  A lattice with no path above -inf gets score -inf, one whose every path is NaN gets NaN,
    invalid lengths (compact: also outside ``compact_hints``) get NaN, all with frames -1.  Deterministic; no host
    synchronisation in the dense layout and, inside ``compact_hints``, in the compact one (CUDA-graph capturable).
    bfloat16 results equal those of the float32 call on the widened logits, and compact results equal those of the
    dense call on the same rows placed in a padded tensor.  Bad values raise ValueError before any launch.

    ``use_hat_loss=True``: the edge weights are the HAT pairs (b, l) of ``rnnt_loss_from_logits(use_hat_loss=True)``,
    bit for bit the loss's, with everything above unchanged (``"regular"`` then equals ``rnnt_align`` on those pairs).
    Needs V >= 2.  The implementation follows k2's ``get_hat_logprobs``; it was not tested against k2 or NeMo."""
    assert isinstance(blank, int)
    assert isinstance(compact, bool)
    kind, lam = _path_type("rnnt_align_from_logits", rnnt_type, delay_penalty, 0.0, compact)
    hat = _use_hat("rnnt_align_from_logits", use_hat_loss, logits)
    with torch.no_grad():
        if compact:
            hints = _hints()
            return _C.rnnt_align_logits_compact(logits, labels, frames_lengths, labels_lengths, blank, hints[0],
                                                hints[1], hat)
        return _C.rnnt_align_logits_dense(logits, labels, frames_lengths, labels_lengths, blank, kind, lam, hat)


def rnnt_align_tdt(logits, labels, frames_lengths, labels_lengths, durations, sigma=0.0, blank=0, compact=False):
    """Viterbi forced alignment on the Token-and-Duration Transducer lattice of ``rnnt_loss_tdt``: the single best
    path, with the frame and the duration of each label, for word timings, segmentation and emission latency.

    Inputs and argument checks are those of ``rnnt_loss_tdt``: dense (N, T, U, V + D) logits, float32 or bfloat16, with
    labels (N, U-1); or ``compact=True``: (STU, V + D) rows in ``joint_pack``'s order with labels
    (sum(labels_lengths),), honouring ``compact_hints``.  durations, sigma and blank as there.  No autograd: the
    outputs are not differentiable and ``logits.requires_grad`` is ignored.

    The lattice, its edges and their weights are ``rnnt_loss_tdt``'s with the same sigma, each log-prob clamped below
    at -1e30 (a masked -inf becomes that finite sentinel).  A path runs from (0, 0) to a terminal blank edge; its score
    is the float32 left fold over its edges in path order, each edge adding its token log-prob and then its duration
    log-prob, ``acc = (acc + lt) + ld``.  The max-plus recurrence adds in that order and so gives the largest such
    score exactly (float32 rounding is monotone).  Ties: the larger candidate wins; on equal values a blank edge beats
    a label edge, and within one kind the shorter duration wins (also for the terminal edge).

    Returns ``(scores, frames, label_durations)``:
      * ``scores`` (N,) float32: the best path's score.
      * ``frames`` int32, dense (N, U-1), compact (sum(labels_lengths),) in the labels' order: frames[n, u] is the frame
        t of the best path's label edge for label u, (t, u) -> (t + d, u + 1).
      * ``label_durations`` int32, the same shape: that edge's duration d, a value of ``durations`` (not an index).
      Both are -1 for u >= labels_lengths[n] and on every lattice without an alignment.

    Lattices without an alignment, in the classes of ``rnnt_loss_tdt`` on the same input: invalid lengths (compact:
    also outside ``compact_hints``, or rows running past STU) or a live label outside [0, V) give score NaN; a NaN or
    +inf in a live row, or a live row whose token or duration logits are all -inf, gives NaN (even for a row no path
    visits); no path above the loss's dead threshold (best score at or below -5e29, e.g. Tn < min(d > 0)) gives -inf.
    Padding rows are never read.  Deterministic; no host synchronisation in the dense layout and, inside
    ``compact_hints``, in the compact one (CUDA-graph capturable); without hints the compact call makes one 16-byte
    device->host copy.  bfloat16 results equal those of the float32 call on the widened logits, and compact results
    equal those of the dense call on the same rows placed in a padded tensor."""
    assert isinstance(compact, bool)
    durations = _tdt_args("rnnt_align_tdt", logits, durations, sigma, blank, compact)
    with torch.no_grad():
        if compact:
            hints = _hints()
            return _C.rnnt_tdt_align_compact(logits, labels, frames_lengths, labels_lengths, list(durations),
                                             float(sigma), blank, hints[0], hints[1])
        return _C.rnnt_tdt_align_dense(logits, labels, frames_lengths, labels_lengths, list(durations), float(sigma),
                                       blank)


def rnnt_align_multiblank(logits, labels, frames_lengths, labels_lengths, big_blank_durations, sigma=0.0, blank=None,
                          compact=False):
    """Viterbi forced alignment on the multi-blank transducer lattice of ``rnnt_loss_multiblank``: the single best
    path, with the frame of each label and how often it takes each blank, for token timings and for how much a trained
    model relies on its big blanks.

    Inputs and argument checks are those of ``rnnt_loss_multiblank``: dense (N, T, U, V) logits, float32 or bfloat16,
    with labels (N, U-1); or ``compact=True``: (STU, V) rows in ``joint_pack``'s order with labels
    (sum(labels_lengths),), honouring ``compact_hints``.  big_blank_durations, sigma and blank as there (blank None:
    V - 1; big blank i in column blank - 1 - i).  No autograd: the outputs are not differentiable and
    ``logits.requires_grad`` is ignored.

    The lattice, its edges and their weights are ``rnnt_loss_multiblank``'s with the same sigma, each weight
    lp = log_softmax(row) - sigma clamped below at -1e30 (a masked -inf becomes that finite sentinel).  A path runs from
    (0, 0) up to and including a terminal edge (the standard blank from (Tn-1, Un-1), or big blank i from
    (Tn-d_i, Un-1)); its score is the float32 left fold ``acc = acc + lp`` over its edges in path order.  The max-plus
    recurrence adds in that order and so gives the largest such score exactly (float32 rounding is monotone).  Ties:
    only a strictly larger candidate replaces the one held, the candidates taken as the standard blank, then the big
    blanks by increasing duration, then the label; so on equal values a blank beats a label and the shorter blank wins
    (also for the terminal edge).  A NaN candidate is never taken.

    Returns ``(scores, frames, blank_counts)``:
      * ``scores`` (N,) float32: the best path's score.
      * ``frames`` int32, dense (N, U-1), compact (sum(labels_lengths),) in the labels' order: frames[n, u] is the
        frame t of the best path's label edge (t, u) -> (t, u+1); non-decreasing, in [0, Tn-1], and -1 for
        u >= labels_lengths[n].
      * ``blank_counts`` (N, 1 + B) int32 in both layouts: column 0 counts the best path's standard-blank edges
        (the terminal edge included), column 1 + i its uses of big blank i; counts[0] + sum_i d_i counts[1+i] = Tn.
      Both are -1 throughout on every lattice without an alignment.

    Lattices without an alignment, in the classes of ``rnnt_loss_multiblank`` on the same input: invalid lengths
    (compact: also outside ``compact_hints``, or rows running past STU) or a live label outside [0, V) give score NaN;
    a NaN or +inf in a live row, or a live row that is all -inf, gives NaN (even for a row no path visits); a best score
    at or below the loss's dead threshold (-5e29) gives -inf, which only masked logits can cause, as the standard blank
    always leaves a path.  Padding rows are never read.  Deterministic; no host synchronisation in the dense layout
    and, inside ``compact_hints``, in the compact one (CUDA-graph capturable); without hints the compact call makes one
    16-byte device->host copy.  bfloat16 results equal those of the float32 call on the widened logits, and compact
    results equal those of the dense call on the same rows placed in a padded tensor."""
    assert isinstance(compact, bool)
    durations, blank = _multiblank_args("rnnt_align_multiblank", logits, big_blank_durations, sigma, blank, compact)
    with torch.no_grad():
        if compact:
            hints = _hints()
            return _C.rnnt_multiblank_align_compact(logits, labels, frames_lengths, labels_lengths, list(durations),
                                                    float(sigma), blank, hints[0], hints[1])
        return _C.rnnt_multiblank_align_dense(logits, labels, frames_lengths, labels_lengths, list(durations),
                                              float(sigma), blank)


__all__ = ["rnnt_loss", "rnnt_align", "rnnt_align_from_logits", "rnnt_align_tdt", "rnnt_align_multiblank", "rnnt_loss_from_logits",
           "rnnt_loss_pruned",
           "rnnt_loss_multiblank", "RNNTLossMultiblank", "RNNTLossMultiblankCompact",
           "RNNTLossPruned", "rnnt_loss_simple", "RNNTLossSimple", "rnnt_loss_tdt", "RNNTLossTDT", "RNNTLossTDTCompact", "joint_pack",
           "JointPack", "RNNTLossFromLogits", "RNNTLossFromLogitsCompact", "RNNTLoss", "RNNTLossGather", "RNNTLossEager",
           "RNNTLossCompact", "compact_hints", "set_lse_mode", "core", "_C", "__version__"]
