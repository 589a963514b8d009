"""GPU: every argument check of the `_C` operator module, one row per condition.

Each row builds a valid call of one entry point from small seeded inputs, breaks exactly one condition (or, for the
rows that pin an order, two) and asserts the first line of the RuntimeError and that no kernel was launched.  A row
whose message is None pins a call that returns today although an argument is out of range, because the empty batch
returns before that check.  The device rows for a second GPU skip on a machine with one; they, and the CPU `lf` / `lg`
rows of rnnt_joint_pack_backward, are built as empty batches, so a binding without the check returns (or reports a
status) without launching anything."""
import pytest
import torch

pytestmark = pytest.mark.gpu

N, T, U, V, S, H = 2, 3, 4, 5, 2, 6


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def _gen():
    return torch.Generator().manual_seed(0)


def _cuda(*ts):
    return [t.cuda() for t in ts]


def _dense(n):
    g = _gen()
    xs = torch.randn(n, T, U, V, generator=g).log_softmax(-1)
    ys = torch.randint(1, V, (n, U - 1), generator=g, dtype=torch.int32)
    xn = torch.full((n,), T, dtype=torch.int32)
    yn = torch.full((n,), U - 1, dtype=torch.int32)
    return _cuda(xs, ys, xn, yn)


def _compact(n):
    g = _gen()
    xn = torch.tensor([3, 2][:n], dtype=torch.int32)
    yn = torch.tensor([2, 1][:n], dtype=torch.int32)
    stu = int((xn * (yn + 1)).sum())
    xs = torch.randn(stu, V, generator=g).log_softmax(-1)
    ys = torch.randint(1, V, (int(yn.sum()),), generator=g, dtype=torch.int32)
    return _cuda(xs, ys, xn, yn)


def _four(xs, ys, xn, yn):
    return dict(xs=xs, ys=ys, xn=xn, yn=yn)


def _pruned(n):
    xs, ys, xn, yn = _dense(n)
    logits = torch.randn(n, T, S, V, generator=_gen()).cuda()
    return dict(xs=logits, ys=ys, xn=xn, yn=yn, ranges=torch.zeros(n, T, dtype=torch.int32, device="cuda"))


def _simple(n):
    _, ys, xn, yn = _dense(n)
    g = _gen()
    am, lm = _cuda(torch.randn(n, T, V, generator=g), torch.randn(n, U, V, generator=g))
    return dict(am=am, lm=lm, ys=ys, xn=xn, yn=yn)


def _joint(n):
    g = _gen()
    f, gg = _cuda(torch.randn(n, T, H, generator=g), torch.randn(n, U, H, generator=g))
    lf, lg = _cuda(torch.tensor([3, 2][:n], dtype=torch.int32), torch.tensor([3, 1][:n], dtype=torch.int32))
    return dict(f=f, g=gg, lf=lf, lg=lg)


def _args(w, entry, n):
    """kwargs of a valid call of `entry` with batch size n."""
    C = w._C
    if entry in ("rnnt_loss", "rnnt_gather_forward", "rnnt_logits_forward", "rnnt_align_dense"):
        return dict(_four(*_dense(n)), blank=0)
    if entry in ("rnnt_loss_dense", "rnnt_loss_fused"):
        return dict(_four(*_dense(n)), blank=0, grad_scale=torch.ones(n, device="cuda"), want_grads=True)
    if entry in ("rnnt_loss_compact", "rnnt_logits_compact_forward", "rnnt_align_compact"):
        return dict(_four(*_compact(n)), blank=0)
    if entry == "rnnt_loss_compact_backward":
        xs, ys, xn, yn = _compact(n)
        _, grads, loc = C.rnnt_loss_compact(xs, ys, xn, yn, 0, 0.0, True)
        cum = torch.cumsum(xn * (yn + 1), 0, dtype=torch.int32)
        return dict(grad_costs=torch.ones(n, device="cuda"), grad_xs=grads, cumSum=cum, loc=loc, V=V, blank=0)
    if entry == "rnnt_rescale_":
        return dict(grads=_dense(n)[0].clone(), grad_out=torch.ones(n, device="cuda"),
                    applied=torch.ones(n, device="cuda"))
    if entry == "rnnt_logits_backward":
        xs, ys, xn, yn = _dense(n)
        _, lse, pg = C.rnnt_logits_forward(xs, ys, xn, yn)
        return dict(xs=xs, lse=lse, pair_grads=pg, ys=ys, grad_out=torch.ones(n, device="cuda"), blank=0)
    if entry == "rnnt_logits_compact_backward":
        xs, ys, xn, yn = _compact(n)
        _, lse, pg, prefix = C.rnnt_logits_compact_forward(xs, ys, xn, yn)
        return dict(xs=xs, lse=lse, pair_grads=pg, ys=ys, xn=xn, yn=yn, prefix=prefix,
                    grad_out=torch.ones(n, device="cuda"), blank=0)
    if entry == "rnnt_logits_pruned_forward":
        return dict(_pruned(n), blank=0)
    if entry == "rnnt_logits_pruned_backward":
        a = _pruned(n)
        _, lse, pg = C.rnnt_logits_pruned_forward(**a)
        return dict(xs=a["xs"], lse=lse, pair_grads=pg, ys=a["ys"], ranges=a["ranges"],
                    grad_out=torch.ones(n, device="cuda"), blank=0)
    if entry == "rnnt_simple_forward":
        return dict(_simple(n), blank=0, want_grads=True, prune_range=2)
    if entry == "rnnt_simple_backward":
        a = _simple(n)
        _, saved, pg, _ = C.rnnt_simple_forward(**a)
        return dict(a, saved=saved, pair_grads=pg, grad_out=torch.ones(n, device="cuda"), blank=0)
    if entry == "rnnt_prune_ranges":
        a = _simple(n)
        pg = C.rnnt_simple_forward(**a)[2]
        return dict(pair_grads=pg, xn=a["xn"], yn=a["yn"], S=2)
    if entry == "rnnt_joint_pack":
        return _joint(n)
    if entry == "rnnt_joint_pack_backward":
        a = _joint(n)
        x, mem_pref = C.rnnt_joint_pack(**a)
        # an empty batch returns the (2,) scratch as mem_pref: take its first n entries
        return dict(dx=torch.ones_like(x), lf=a["lf"], lg=a["lg"], mem_pref=mem_pref[:n], T=T, U1=U)
    if entry == "rnnt_gather_backward":
        xs, ys, xn, yn = _dense(n)
        pg = C.rnnt_gather_forward(xs, ys, xn, yn)[1]
        return dict(pair_grads=pg, ys=ys, grad_out=torch.ones(n, device="cuda"), V=V, blank=0, accumulate=True, yn=yn)
    raise KeyError(entry)


ENTRIES = ["rnnt_loss", "rnnt_loss_compact", "rnnt_loss_compact_backward", "rnnt_loss_dense", "rnnt_loss_fused",
           "rnnt_rescale_", "rnnt_gather_forward", "rnnt_gather_backward", "rnnt_logits_forward",
           "rnnt_logits_backward", "rnnt_logits_compact_forward", "rnnt_logits_compact_backward",
           "rnnt_logits_pruned_forward", "rnnt_logits_pruned_backward", "rnnt_simple_forward", "rnnt_simple_backward",
           "rnnt_prune_ranges", "rnnt_joint_pack", "rnnt_joint_pack_backward", "rnnt_align_dense",
           "rnnt_align_compact"]


# ---- how an argument is broken -----------------------------------------------------------------------------------

def _breaker(name, fn):
    fn.__name__ = name
    return fn


def _strided(t):
    buf = torch.zeros(*t.shape, 2, dtype=t.dtype, device=t.device)
    buf[..., 0] = t
    return buf[..., 0]


NC = _breaker("strided", _strided)                                        # same values, not contiguous
CPU = _breaker("cpu", lambda t: t.cpu())
DEV1 = _breaker("cuda1", lambda t: t.to("cuda:1"))
F64 = _breaker("f64", lambda t: t.double())
BF16 = _breaker("bf16", lambda t: t.bfloat16())
I64 = _breaker("i64", lambda t: t.long())
I32 = _breaker("i32", lambda t: t.int())
ADD_DIM = _breaker("add_dim", lambda t: t.unsqueeze(0).contiguous())
FLAT = _breaker("flat", lambda t: t.reshape(-1))
LAST0 = _breaker("drop_last_dim", lambda t: t[..., 0].contiguous())


def SHORT(dim):
    """One element fewer along `dim`."""
    return _breaker("short%d" % dim, lambda t: t.narrow(dim, 0, t.size(dim) - 1).contiguous())


ROWS = []


def row(entry, msg, n=N, **change):
    ROWS.append((entry, n, change, msg))


# ---- check4: contiguity, then dtypes, then device, as in the reference; then the device of xs ----------------------

CHECK4 = {"rnnt_loss": False, "rnnt_loss_compact": False, "rnnt_loss_dense": False, "rnnt_loss_fused": True,
          "rnnt_gather_forward": False, "rnnt_logits_forward": True, "rnnt_logits_compact_forward": True,
          "rnnt_logits_pruned_forward": True, "rnnt_align_dense": True, "rnnt_align_compact": True}
for e, bf16_ok in CHECK4.items():
    for a in ("xs", "ys", "xn", "yn"):
        row(e, "%s must be contiguous" % a, **{a: NC})
        row(e, "%s must be located in the CUDA" % a, **{a: CPU})
    for a in ("ys", "xn", "yn"):
        row(e, "%s must be a Int tensor" % a, **{a: I64})
        row(e, "%s must be on the device of xs" % a, n=0, **{a: DEV1})
    row(e, "xs must be a Float tensor", xs=F64)
    if not bf16_ok:
        row(e, "xs must be a Float tensor", xs=BF16)
    # the phases' order (rnnt_loss_fused checks the device of xs before check4)
    cpu_xs = "xs must be located in the CUDA" if e == "rnnt_loss_fused" else None
    row(e, cpu_xs or "ys must be a Int tensor", xs=CPU, ys=I64)
    row(e, "ys must be contiguous", xs=F64, ys=NC)
    row(e, cpu_xs or "yn must be a Int tensor", xs=CPU, yn=I64)
    row(e, "yn must be located in the CUDA", n=0, ys=DEV1, yn=CPU)

# ---- the dense shapes, blank and the empty batch ----------------------------------------------------------------

for e in ("rnnt_loss", "rnnt_loss_dense", "rnnt_loss_fused", "rnnt_gather_forward", "rnnt_logits_forward",
          "rnnt_align_dense"):
    row(e, "xs must have 4 dimensions", xs=LAST0)
    row(e, "xn shape must be equal (N,)", xn=SHORT(0))
    row(e, "yn shape must be equal (N,)", yn=SHORT(0))
    row(e, "ys shape (N, U-1) mismatched with xs (N, T, U, V)", ys=FLAT)
    row(e, "ys shape (N, U-1) mismatched with xs (N, T, U, V)", ys=SHORT(1))
for e in ("rnnt_loss", "rnnt_loss_dense", "rnnt_loss_fused"):
    row(e, "blank must be in [0, V) (or -1 for the gathered layout)", blank=V)
    row(e, None, n=0, blank=99)                                      # the empty batch returns before blank is read
for e in ("rnnt_loss", "rnnt_loss_dense"):
    row(e, "blank must be in [0, V) (or -1 for the gathered layout)", blank=-2)
    row(e, "xs must have values only for blank and label", blank=-1)
for e in ("rnnt_loss_dense", "rnnt_loss_fused"):
    for b in (NC, F64, CPU, SHORT(0)):
        row(e, "grad_scale must be a contiguous Float tensor of shape (N,) on the device of xs", grad_scale=b)
row("rnnt_loss_fused", "rnnt_loss_fused takes the dense (N,T,U,V) layout", blank=-1)
row("rnnt_loss_fused", "rnnt_loss_fused takes the dense (N,T,U,V) layout", blank=-1, xs=CPU)
row("rnnt_loss_fused", "xs must be located in the CUDA", xs=_breaker("strided_cpu", lambda t: NC(t.cpu())))
row("rnnt_loss_fused", "bfloat16 xs: dense (N,T,U,V) layout with gradients only", xs=BF16, want_grads=False)
row("rnnt_loss_fused", None, n=0, xs=BF16, want_grads=False)
for e in ("rnnt_gather_forward", "rnnt_logits_forward", "rnnt_align_dense", "rnnt_logits_pruned_forward",
          "rnnt_loss_compact", "rnnt_logits_compact_forward", "rnnt_align_compact"):
    row(e, "blank must be in [0, V)", blank=V)
    row(e, "blank must be in [0, V)", blank=-1)
    row(e, "blank must be in [0, V)", n=0, blank=99)                 # blank is checked before the empty batch returns

# ---- the compact shapes -------------------------------------------------------------------------------------------

for e in ("rnnt_loss_compact", "rnnt_logits_compact_forward", "rnnt_align_compact"):
    row(e, "xs must have 2 dimensions", xs=ADD_DIM)
    row(e, "xn and yn shape must be equal (N,)", xn=ADD_DIM)
    row(e, "xn and yn shape must be equal (N,)", yn=ADD_DIM)
    row(e, "xn and yn shape must be equal (N,)", xn=SHORT(0))

# ---- rnnt_loss_compact_backward: the reference's phases, then the device of grad_cost -----------------------------

e = "rnnt_loss_compact_backward"
for a, dt in (("grad_costs", F64), ("grad_xs", F64), ("loc", I32)):
    name = {"grad_costs": "grad_cost"}.get(a, a)
    row(e, "%s must be contiguous" % name, **{a: NC})
    row(e, "%s must be a %s tensor" % (name, "Long" if a == "loc" else "Float"), **{a: dt})
    row(e, "%s must be located in the CUDA" % name, **{a: CPU})
row(e, "cum_lens must be located in the CUDA", cumSum=CPU)
for a, name in (("grad_xs", "grad_xs"), ("cumSum", "cum_lens"), ("loc", "loc")):
    row(e, "%s must be on the device of grad_cost" % name, n=0, **{a: DEV1})
row(e, "grad_cost must have 1 dimensions", grad_costs=ADD_DIM)
row(e, "grad must have 2 dimensions", grad_xs=FLAT)
row(e, "grad and loc must be equal in dim=0", loc=SHORT(0))
for b in (NC, I64, SHORT(0)):
    row(e, "cum_lens must be a contiguous Int tensor of shape (N,)", cumSum=b)
row(e, "grad must have shape (STU, 2)", grad_xs=SHORT(1))
row(e, "blank must be in [0, V)", blank=V)
row(e, "blank must be in [0, V)", blank=-1)
row(e, "loc must be a Long tensor", grad_xs=CPU, loc=I32)
row(e, "grad_xs must be contiguous", grad_costs=F64, grad_xs=NC)

# ---- rnnt_rescale_ ----------------------------------------------------------------------------------------------

e = "rnnt_rescale_"
for b in (NC, F64, CPU, _breaker("scalar", lambda t: t.flatten()[0].clone())):
    row(e, "grads must be a contiguous CUDA Float (or BFloat16) tensor", grads=b)
for b in (NC, F64, CPU, _breaker("three", lambda t: torch.ones(3, device=t.device))):
    row(e, "grad_out must be a contiguous Float tensor with N elements (or one) on the device of grads", grad_out=b)
    row(e, "applied must be a contiguous Float tensor of shape (N,) on the device of grads", applied=b)

# ---- tensors checked as a whole: contiguous, dtype, device, shape, one message ------------------------------------

FLOAT = (NC, F64, CPU)
INT = (NC, I64, CPU)
LONG = (NC, I32, CPU)


def whole(entry, arg, msg, breaks):
    for b in breaks:
        row(entry, msg, **{arg: b})


for e, xs_msg, lse_msg, pg_msg in (
        ("rnnt_logits_backward", "xs must be a contiguous CUDA Float tensor of shape (N, T, U, V)",
         "lse must be a contiguous Float tensor of shape (N, T, U) on the device of xs",
         "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of xs"),
        ("rnnt_logits_compact_backward", "xs must be a contiguous CUDA Float tensor of shape (STU, V)",
         "lse must be a contiguous Float tensor of shape (STU,) on the device of xs",
         "pair_grads must be a contiguous Float tensor of shape (STU, 2) on the device of xs"),
        ("rnnt_logits_pruned_backward", "xs must be a contiguous CUDA Float tensor of shape (N, T, S, V)",
         "lse must be a contiguous Float tensor of shape (N, T, S) on the device of xs",
         "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of xs")):
    whole(e, "xs", xs_msg, FLOAT + (ADD_DIM,))
    whole(e, "lse", lse_msg, FLOAT + (SHORT(0),))
    whole(e, "pair_grads", pg_msg, FLOAT + (SHORT(0),))
    whole(e, "grad_out", "grad_out must be a contiguous Float tensor of shape (N,)", FLOAT + (SHORT(0),))
    row(e, "blank must be in [0, V)", blank=V)
    row(e, "blank must be in [0, V)", blank=-1)
whole("rnnt_logits_backward", "ys", "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs",
      INT + (FLAT, SHORT(0), SHORT(1)))
whole("rnnt_logits_compact_backward", "ys", "ys must be a contiguous Int tensor on the device of xs", INT)
for a in ("xn", "yn"):
    whole("rnnt_logits_compact_backward", a, "xn and yn must be contiguous Int tensors of shape (N,) on the device of xs",
          INT)
row("rnnt_logits_compact_backward", "xn and yn must be contiguous Int tensors of shape (N,) on the device of xs",
    yn=SHORT(0))
whole("rnnt_logits_compact_backward", "prefix",
      "prefix must be a contiguous Long tensor of shape (2N,) on the device of xs", LONG + (SHORT(0),))
whole("rnnt_logits_pruned_backward", "ys", "ys must be a contiguous Int tensor of shape (N, U-1) on the device of xs",
      INT + (FLAT, SHORT(0)))
RANGES = "ranges must be a contiguous Int tensor of shape (N, T) on the device of xs"
for e in ("rnnt_logits_pruned_forward", "rnnt_logits_pruned_backward"):
    whole(e, "ranges", RANGES, INT + (FLAT, SHORT(0), SHORT(1)))

e = "rnnt_logits_pruned_forward"
row(e, "xs must have 4 dimensions", xs=LAST0)
row(e, "xn shape must be equal (N,)", xn=SHORT(0))
row(e, "yn shape must be equal (N,)", yn=SHORT(0))
row(e, "ys shape must be (N, U-1)", ys=FLAT)
row(e, "ys shape must be (N, U-1)", ys=SHORT(0))

# ---- the simple loss and its ranges -------------------------------------------------------------------------------

for e in ("rnnt_simple_forward", "rnnt_simple_backward"):
    for a in ("am", "lm"):
        row(e, "am and lm must be float32 tensors (the simple loss does not take bfloat16)", **{a: F64})
        row(e, "am and lm must be float32 tensors (the simple loss does not take bfloat16)", **{a: BF16})
        row(e, "am and lm must be contiguous CUDA tensors on one device", **{a: NC})
        row(e, "am and lm must be contiguous CUDA tensors on one device", **{a: CPU})
        row(e, "am must be (N, T, V) and lm (N, U, V)", **{a: LAST0})
    row(e, "am must be (N, T, V) and lm (N, U, V)", lm=SHORT(0))
    row(e, "am must be (N, T, V) and lm (N, U, V)", lm=SHORT(2))
    whole(e, "ys", "ys must be a contiguous Int tensor of shape (N, U-1) on the device of am",
          INT + (FLAT, SHORT(0), SHORT(1)))
    for a in ("xn", "yn"):
        whole(e, a, "xn and yn must be contiguous Int tensors of shape (N,) on the device of am", INT + (SHORT(0),))
    row(e, "blank must be in [0, V)", blank=V)
    row(e, "blank must be in [0, V)", blank=-1)
row("rnnt_simple_forward", "prune_range must be an int >= 2", prune_range=1)
row("rnnt_simple_forward", "prune_range must be an int >= 2", prune_range=-1)
e = "rnnt_simple_backward"
whole(e, "saved", "saved must be the simple forward's contiguous Float tensor on the device of am", FLOAT + (SHORT(0),))
whole(e, "pair_grads", "pair_grads must be a contiguous Float tensor of shape (N, T, U, 2) on the device of am",
      FLOAT + (SHORT(0),))
whole(e, "grad_out", "grad_out must be a contiguous Float tensor of shape (N,)", FLOAT + (SHORT(0),))

e = "rnnt_prune_ranges"
whole(e, "pair_grads", "pair_grads must be a contiguous CUDA Float tensor of shape (N, T, U, 2)",
      FLOAT + (LAST0, SHORT(3)))
for a in ("xn", "yn"):
    whole(e, a, "xn and yn must be contiguous Int tensors of shape (N,) on the device of pair_grads", INT + (SHORT(0),))
row(e, "prune_range must be an int >= 2", S=1)

# ---- gather backward --------------------------------------------------------------------------------------------

e = "rnnt_gather_backward"
whole(e, "pair_grads", "pair_grads must be a contiguous CUDA Float tensor of shape (N, T, U, 2)",
      FLOAT + (LAST0, SHORT(3)))
whole(e, "ys", "ys must be a contiguous Int tensor on the device of pair_grads", INT)
whole(e, "grad_out", "grad_out must be a contiguous Float tensor of shape (N,)", FLOAT + (SHORT(0),))
whole(e, "ys", "ys shape (N, U-1) mismatched", (FLAT, SHORT(0), SHORT(1)))
row(e, "blank must be in [0, V)", blank=V)
row(e, "blank must be in [0, V)", blank=-1)
whole(e, "yn", "yn must be a contiguous Int tensor of shape (N,) on the device of pair_grads", INT + (SHORT(0),))

# ---- joint packing ----------------------------------------------------------------------------------------------

e = "rnnt_joint_pack"
for a in ("f", "g", "lf", "lg"):
    row(e, "inputs must be contiguous", **{a: NC})
    row(e, "f, g, lf, lg must be on the same CUDA device", **{a: CPU})
for a in ("f", "g"):
    row(e, "f and g must be Float tensors", **{a: F64})
    row(e, "f must be (N, T, H) and g (N, U+1, H)", **{a: LAST0})
row(e, "f must be (N, T, H) and g (N, U+1, H)", g=SHORT(0))
row(e, "f must be (N, T, H) and g (N, U+1, H)", g=SHORT(2))
for a in ("lf", "lg"):
    row(e, "lf and lg must be Int tensors", **{a: I64})
    row(e, "lf and lg must have N elements", **{a: SHORT(0)})

e = "rnnt_joint_pack_backward"
whole(e, "dx", "dx must be a contiguous CUDA Float tensor of shape (STU, H)", FLOAT + (FLAT,))
whole(e, "mem_pref", "mem_pref must be a contiguous Long tensor on the device of dx", LONG)
for a in ("lf", "lg"):
    whole(e, a, "lf and lg must be contiguous Int tensors with N elements", (NC, I64, SHORT(0)))
    row(e, "lf and lg must be on the device of dx", n=0, **{a: CPU})
    row(e, "lf and lg must be on the device of dx", n=0, **{a: DEV1})


def _row_id(r):
    entry, n, change, _ = r
    parts = ["%s=%s" % (k, getattr(v, "__name__", v)) for k, v in change.items()]
    return "%s:%s%s" % (entry, ",".join(parts), ":N=0" if n == 0 else "")


def _param(r):
    two = any(v is DEV1 for v in r[2].values())
    marks = [pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second CUDA device")] if two else []
    return pytest.param(*r, id=_row_id(r), marks=marks)


@pytest.mark.parametrize("entry", ENTRIES)
def test_valid_call(w, entry):
    """The unbroken call of every entry point succeeds, at N = 2 and at the N = 0 of the empty-batch rows, so each
    row breaks only what it names.  (rnnt_joint_pack_backward's empty batch is refused by the C ABI, status 5: its
    rows are refused by the binding before that.)"""
    empty = {r[0] for r in ROWS if r[1] == 0} - {"rnnt_joint_pack_backward"}
    for n in (N, 0) if entry in empty else (N,):
        getattr(w._C, entry)(**_args(w, entry, n))
    torch.cuda.synchronize()


def test_every_entry_point_has_rows():
    assert {r[0] for r in ROWS} == set(ENTRIES)


@pytest.mark.parametrize("entry,n,change,msg", [_param(r) for r in ROWS])
def test_check(w, entry, n, change, msg):
    kw = _args(w, entry, n)
    for k, b in change.items():
        kw[k] = b(kw[k]) if callable(b) else b
    torch.cuda.synchronize()
    before = w._C.launch_count()
    if msg is None:
        getattr(w._C, entry)(**kw)
    else:
        with pytest.raises(RuntimeError) as e:
            getattr(w._C, entry)(**kw)
        assert str(e.value).splitlines()[0] == msg
    assert w._C.launch_count() == before, "a kernel was launched before the arguments were refused"
