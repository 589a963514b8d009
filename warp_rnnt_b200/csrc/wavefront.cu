// wavefront.cu -- general (any-size) path: prefix sums, log-prob gather, the alpha/beta wavefront
// and the (cells,2) gradient kernel; and the Viterbi alignment (k_align), the alpha wavefront in max-plus form.
//
// What it replaces in the reference (1ytic/warp-rnnt):
//   k_prefix      : host-side cumsum + 4 .item() syncs        pytorch_binding/binding.cpp:132-158
//   k_gather      : kernel_fill_gather                        core_compact.cu:403-436
//                   python-level gather (index tensor + torch.gather)   warp_rnnt/__init__.py:118-128
//   k_wavefront   : kernel_warp_alphas / kernel_warp_betas + the counts scheduler
//                   core.cu:41-258, core_gather.cu:37-246, core_compact.cu:29-269
//                   kernel_fill_costs (+ mismatch guard)      core.cu:334-370, core_compact.cu:347-358
//   k_grads_pairs : kernel_grads_blank / kernel_grads_label   core.cu:260-332, core_compact.cu:271-345
//
// Design (not a port): one CTA per (lattice, direction); alpha and beta CTAs of a lattice form a
// 2-CTA cluster and meet on a cluster barrier for the cost / mismatch guard.  Inside a CTA lane l
// of warp w owns lattice column 32w+l and walks the anti-diagonals: one __shfl_up per step moves
// the cell value to the right-hand neighbour, warps hand their boundary column to the next warp
// through a shared-memory ring (tagged 64-bit slots, no barrier on the dependent chain).  The
// reference instead tiles the lattice into 32x1 blocks ordered by global atomics + __threadfence.
#include "common.cuh"
#include "kernels.cuh"

namespace rnnt {

// ------------------------------------------------------------------------------------------
// k_prefix: exclusive prefix sums of xn*(yn+1) and yn (int64), totals for host validation.
// One block; N is small (batch size).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_prefix(const int *__restrict__ xn, const int *__restrict__ yn, int N,
                                                  int64_t *__restrict__ mem_pref, int64_t *__restrict__ lab_pref,
                                                  int *__restrict__ totals) {
    __shared__ int64_t s_mem[32], s_lab[32];
    __shared__ int s_tm[32], s_um[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (N + blockDim.x - 1) / blockDim.x;
    const int lo = min(tid * per, N), hi = min(lo + per, N);
    int64_t sm = 0, sl = 0;
    int tm = 0, um = 0;
    for (int i = lo; i < hi; ++i) {
        const int x = xn[i], y = yn[i];
        sm += (int64_t)x * (y + 1);
        sl += y;
        tm = max(tm, x);
        um = max(um, y + 1);
    }
    // inclusive warp scan of (sm, sl), warp max of (tm, um)
    int64_t im = sm, il = sl;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int64_t a = __shfl_up_sync(0xffffffffu, im, o);
        int64_t b = __shfl_up_sync(0xffffffffu, il, o);
        if (lane >= o) { im += a; il += b; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tm = max(tm, __shfl_xor_sync(0xffffffffu, tm, o));
        um = max(um, __shfl_xor_sync(0xffffffffu, um, o));
    }
    if (lane == 31) { s_mem[warp] = im; s_lab[warp] = il; }
    if (lane == 0) { s_tm[warp] = tm; s_um[warp] = um; }
    __syncthreads();
    if (warp == 0) {
        int64_t a = s_mem[lane], b = s_lab[lane];
        const int nw = blockDim.x >> 5;
        if (lane >= nw) { a = 0; b = 0; }
        int64_t ia = a, ib = b;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int64_t x = __shfl_up_sync(0xffffffffu, ia, o);
            int64_t y = __shfl_up_sync(0xffffffffu, ib, o);
            if (lane >= o) { ia += x; ib += y; }
        }
        s_mem[lane] = ia - a;  // exclusive over warps
        s_lab[lane] = ib - b;
        int t2 = lane < nw ? s_tm[lane] : 0, u2 = lane < nw ? s_um[lane] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            t2 = max(t2, __shfl_xor_sync(0xffffffffu, t2, o));
            u2 = max(u2, __shfl_xor_sync(0xffffffffu, u2, o));
        }
        if (lane == 31 && totals) {
            totals[0] = (int)min(ia, (int64_t)INT32_MAX);
            totals[1] = (int)min(ib, (int64_t)INT32_MAX);
            totals[2] = t2;
            totals[3] = u2;
        }
    }
    __syncthreads();
    int64_t rm = s_mem[warp] + (im - sm), rl = s_lab[warp] + (il - sl);  // exclusive prefix of this thread
    for (int i = lo; i < hi; ++i) {
        mem_pref[i] = rm;
        lab_pref[i] = rl;
        rm += (int64_t)xn[i] * (yn[i] + 1);
        rl += yn[i];
    }
}

// ------------------------------------------------------------------------------------------
// k_gather: pairs[cell] = (lp[cell, blank], lp[cell, label(u)]) for valid cells; optional loc.
// grid (gx, N); every thread handles kIlp cells with all loads issued before the stores.
// ------------------------------------------------------------------------------------------
constexpr int kGatherThreads = 256;
constexpr int kGatherIlp = 4;

template <typename IO>
__global__ void __launch_bounds__(kGatherThreads)
k_gather(Problem p, const IO *__restrict__ lp, const int *__restrict__ labels, int V, int blank,
         float2 *__restrict__ pairs, int64_t *__restrict__ loc) {
    const int n = blockIdx.y;
    const Lattice L = get_lattice(p, n);
    if (!L.ok) return;
    const int cells = p.compact ? L.Tn * L.Un : L.Tn * L.stride;  // dense: rows [0,Tn) incl. padded columns
    for (int c0 = (blockIdx.x * kGatherThreads) * kGatherIlp; c0 < cells; c0 += gridDim.x * kGatherThreads * kGatherIlp) {
        float vb[kGatherIlp], vl[kGatherIlp];
        int lab[kGatherIlp];
        int64_t cell[kGatherIlp];
        bool ok[kGatherIlp];
#pragma unroll
        for (int k = 0; k < kGatherIlp; ++k) {
            const int r = c0 + k * kGatherThreads + threadIdx.x;
            ok[k] = r < cells;
            const int t = ok[k] ? r / L.stride : 0;
            const int u = ok[k] ? r - t * L.stride : 0;
            ok[k] = ok[k] && (u < L.Un);
            cell[k] = L.base + r;
            // the last column has no label transition; the reference's compact gather stores the
            // blank there (core_compact.cu:424-431)
            lab[k] = (ok[k] && u < L.Un - 1) ? labels[L.lab_base + u] : blank;
        }
#pragma unroll
        for (int k = 0; k < kGatherIlp; ++k) {
            if (ok[k]) {
                const IO *row = lp + cell[k] * (int64_t)V;
                vb[k] = io_load<IO>(row + blank);
                vl[k] = io_load<IO>(row + lab[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < kGatherIlp; ++k) {
            if (ok[k]) {
                pairs[cell[k]] = make_float2(vb[k], vl[k]);
                if (loc) loc[cell[k]] = lab[k];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// k_wavefront
// ------------------------------------------------------------------------------------------
// kPrefetch (template parameter PF): steps of log-prob prefetch = unroll factor of the recurrence loop

struct __align__(8) Slot { float val; int row; };

// shared-space (32-bit) addresses, computed once per sweep: a generic pointer costs an address-space conversion
// (S2UR + ULEA in a cluster launch) at every access, ~10 of the loop's instructions per step
__device__ __forceinline__ Slot ld_slot_s(uint32_t a) {
    Slot s;
    asm volatile("ld.volatile.shared.v2.b32 {%0, %1}, [%2];" : "=f"(s.val), "=r"(s.row) : "r"(a) : "memory");
    return s;
}
__device__ __forceinline__ void st_slot_s(uint32_t a, float v, int row) {
    asm volatile("st.volatile.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "f"(v), "r"(row) : "memory");
}
__device__ __forceinline__ int ld_vol_s32_s(uint32_t a) {
    int v;
    asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void st_vol_s32_s(uint32_t a, int v) {
    asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ Slot ld_slot(const Slot *p) {
    Slot s;
    asm volatile("ld.volatile.shared.v2.b32 {%0, %1}, [%2];"
                 : "=f"(s.val), "=r"(s.row)
                 : "r"((uint32_t)__cvta_generic_to_shared(p))
                 : "memory");
    return s;
}
__device__ __forceinline__ void st_slot(Slot *p, float v, int row) {
    asm volatile("st.volatile.shared.v2.b32 [%0], {%1, %2};" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "f"(v),
                 "r"(row)
                 : "memory");
}
__device__ __forceinline__ int ld_vol_s32(const int *p) {
    int v;
    asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
    return v;
}
__device__ __forceinline__ void st_vol_s32(int *p, int v) {
    asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}

// Predicated global loads whose destination register is written by the load itself.
__device__ __forceinline__ float ldg_nc_pred(const float *p, bool pred, float dflt) {
    float v;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %2, 0;\n\tmov.f32 %0, %3;\n\t@p ld.global.nc.f32 %0, [%1];\n\t}"
                 : "=f"(v)
                 : "l"(p), "r"((int)pred), "f"(dflt));
    return v;
}
__device__ __forceinline__ float ldg_cg_pred(const float *p, bool pred, float dflt) {
    float v;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %2, 0;\n\tmov.f32 %0, %3;\n\t@p ld.global.cg.f32 %0, [%1];\n\t}"
                 : "=f"(v)
                 : "l"(p), "r"((int)pred), "f"(dflt)
                 : "memory");
    return v;
}

// Where lane 0 of a warp gets its left-hand neighbour column from.
enum LeftSrc { kLeftNone = 0,   // lattice column 0: no left neighbour
               kLeftRing = 1,   // previous warp of this CTA, through the shared-memory ring
               kLeftMem = 2 };  // global memory: previous column pass (U > 32*nwarps), or -- with
                                // `override` -- the pre-computed column 0 of the exact mode

// Per-warp state of one sweep over the warp's 32 columns.
struct Sweep {
    const float2 *pr;   // pairs of this lattice
    float *o;           // alpha or beta of this lattice
    Slot *ring_in, *ring_out;
    int *cons_self, *cons_next;
    int Tn, Un, st, T1, U1;
    int j, lane;
    int nsteps, ring_mask;
    bool col_ok, publish, backpressure, override0;
    uint32_t *dec;      // kMax: this warp's decision words, one per step (word s = the warp's bits at step s)
};

// "Minus infinity" that stays finite: cells outside the lattice carry kBig (common.cuh) so that the one
// uniform step below needs no per-lane control flow.  LSE(kBig, kBig) == kBig (+ln 2, absorbed) and
// kBig + (a finite log-prob) stays ~kBig without ever producing inf - inf.  LSE(x, kBig) == x exactly, in
// every LSE flavour, only while x is well above kBig: for x = -inf, or any x at or below about -1e30, the
// sentinel wins and the result is ~kBig.  Row 0 of alpha and the last row of beta, which the reference
// computes as plain sums, therefore hold ~kBig where the reference has -inf, and a lattice with no alignment
// of finite log-probability ends with beta[0,0] ~ kBig (or NaN) instead of -inf / NaN.  The epilogue
// (k_wavefront) and the gradient kernels map that to the reference's classes: lattice_dead, common.cuh.

// One direction of one lattice.  "Primed" coordinates (i,j): alpha uses (t,u); beta uses
// (Tn-1-t, Un-1-u), so both are the same recurrence
//   val[i,j] = LSE(val[i-1,j] + wB(i,j), val[i,j-1] + wL(i,j)),  val[0,0] = init
// alpha: wB = blank[i-1,j], wL = label[i,j-1], init 0          (core.cu:80-134)
// beta : wB = blank[t,u],   wL = label[t,u] at the own cell, init = blank[T-1,U-1]  (core.cu:171-239)
// Lane l of the warp owns column j and at step s works on row i = s - l.  Edge rules are encoded
// in the operands instead of branches:
//   row 0     : val starts at kBig          -> skip term vanishes, v = emit        (core.cu:80-90)
//   column 0  : wL = kBig for that lane     -> emit term vanishes, v = skip        (core.cu:92-110)
//   cell (0,0): val starts at 0 with wB(0,0) = 0 (alpha) / blank[T-1,U-1] (beta)   (core.cu:64-66,171-173)
//   i < 0     : wL = kBig, wB = 0           -> val stays kBig until the lane's first row
//   i >= Tn   : results are garbage that no in-lattice cell ever reads; stores are masked.
template <int KIND, bool BETA, int SRC, int PF>
__device__ __forceinline__ float sweep_warp(const Sweep &S) {
    constexpr int kPrefetch = PF;
    const int lane = S.lane, j = S.j, Tn = S.Tn, st = S.st, T1 = S.T1, U1 = S.U1;
    const unsigned rows = S.col_ok ? (unsigned)Tn : 0u;    // (unsigned)i < rows  <=>  cell (i,j) is in the lattice
    const bool first_col = (j == 0);
    float val = first_col ? 0.0f : kBig;
    float last = val;         // value of this lane's last in-lattice row
    int cons_seen = 0;        // producer-side cache of the consumer's progress counter
    Slot pre;                 // consumer: ring slot for the next row, loaded one step ahead
    pre.val = 0.0f;
    pre.row = -2;

    // own cell index at step s is c0 + s*ds (64-bit): alpha walks down, beta walks up
    const int64_t ds = BETA ? -(int64_t)st : (int64_t)st;
    const int64_t c0 = BETA ? ((int64_t)(T1 + lane) * st + (U1 - j)) : (-(int64_t)lane * st + j);
    // memory-resident left boundary / column-0 override (lane 0 only)
    const int64_t bcol = S.override0 ? 0 : (BETA ? 1 : -1);
    const bool mem_lane = (SRC == kLeftMem) && lane == 0;

    float wb[kPrefetch], wl[kPrefetch], bnd[kPrefetch];

    // operands of step s into prefetch slot k.  Predicated loads that write the destination
    // register directly (a select after the load would make the prefetch wait for its own data).
    // fetch() is called for s = 0, 1, 2, ... in order: the cell pointers run along (two 64-bit adds per step instead of
    // a 64-bit multiply-add and the pointer arithmetic per load)
    const float *cell = reinterpret_cast<const float *>(S.pr + c0);
    const float *bcell = S.o + c0 + bcol;
    auto fetch = [&](int k, int s) {
        const int i = s - lane;
        const bool in = (unsigned)i < rows;
        if (BETA) {
            wb[k] = ldg_nc_pred(cell, in, 0.0f);
            wl[k] = ldg_nc_pred(cell + 1, in && !first_col, (i < 0 || first_col) ? kBig : 0.0f);
        } else {
            wb[k] = ldg_nc_pred(cell - 2 * (int64_t)st, in && i >= 1, 0.0f);
            wl[k] = ldg_nc_pred(cell - 1, in && !first_col, (i < 0 || first_col) ? kBig : 0.0f);
        }
        if (SRC == kLeftMem) {
            bnd[k] = ldg_cg_pred(bcell, in && mem_lane && (!S.override0 || i >= 1), kBig);
            bcell += ds;
        }
        cell += 2 * ds;
    };

    const uint32_t a_in = (uint32_t)__cvta_generic_to_shared(S.ring_in), a_out = (uint32_t)__cvta_generic_to_shared(S.ring_out);
    const uint32_t a_cself = (uint32_t)__cvta_generic_to_shared(S.cons_self), a_cnext = (uint32_t)__cvta_generic_to_shared(S.cons_next);
    // consumer side of the ring: value of the left neighbour column at row `row` (warp-uniform call)
    auto ring_get = [&](int row) -> float {
        while (pre.row != row) pre = ld_slot_s(a_in + 8u * (uint32_t)(row & S.ring_mask));
        const float v = pre.val;
        if (S.backpressure && lane == 0) st_vol_s32_s(a_cself, row + 1);
        pre = ld_slot_s(a_in + 8u * (uint32_t)((row + 1) & S.ring_mask));   // next row, off the dependent chain
        return v;
    };
    // producer side: lane 31 hands row `row` of its column to the next warp (warp-uniform call)
    auto ring_put = [&](int row, float v) {
        if (S.backpressure && row - S.ring_mask - 1 >= cons_seen) {
            int c = ld_vol_s32_s(a_cnext);
            while (row - S.ring_mask - 1 >= c) c = ld_vol_s32_s(a_cnext);
            cons_seen = c;
        }
        if (lane == 31) st_slot_s(a_out + 8u * (uint32_t)(row & S.ring_mask), v, row);
    };

#pragma unroll
    for (int k = 0; k < kPrefetch; ++k) fetch(k, k);

    float *op = S.o + c0;
    for (int s0 = 0; s0 < S.nsteps; s0 += kPrefetch) {
#pragma unroll
        for (int k = 0; k < kPrefetch; ++k) {
            const int s = s0 + k;                               // steps past nsteps are harmless no-ops
            float left = __shfl_up_sync(0xffffffffu, val, 1);
            if (SRC == kLeftRing) {
                if (s < Tn) {                                   // warp-uniform
                    const float b = ring_get(s);
                    if (lane == 0) left = b;
                }
            } else if (SRC == kLeftMem) {
                if (lane == 0) left = bnd[k];
            }
            const float skip = val + wb[k];
            const float emit = left + wl[k];
            float v;
            if constexpr (KIND == kMax) {
                // max-plus step: the label predecessor iff it is larger or the blank one is NaN (a NaN candidate loses
                // to any number, a tie goes to the blank edge); row 0 and column 0 take their one predecessor as is,
                // so the kBig operands of the border never reach a real cell
                bool bit = (emit > skip) || isnan(skip);
                bit = (bit || s == lane) && !first_col;
                v = bit ? emit : skip;
                const unsigned word = __ballot_sync(0xffffffffu, bit);
                if (lane == 0 && s < S.nsteps) S.dec[s] = word;
            } else {
                v = lse<KIND>(skip, emit);
            }
            if (SRC == kLeftMem) {
                if (S.override0 && lane == 0 && s >= 1) v = bnd[k];   // column 0 from the scan pre-pass
            }
            val = v;
            if ((unsigned)(s - lane) < rows) {
                *op = v;
                last = v;
            }
            op += ds;
            if (S.publish && (unsigned)(s - 31) < (unsigned)Tn) ring_put(s - 31, v);   // warp-uniform
            fetch(k, s + kPrefetch);                            // rolling prefetch, kPrefetch steps ahead
        }
    }
    return last;
}

// kMax (alpha only): dec = the lattice's decision words, column block w (lattice columns 32w .. 32w+31) at
// dec + w * dec_stride; word s of a block holds bit u%32 of cell (t = s - u%32, u), 1 = the label predecessor.
template <int KIND, bool BETA, int PF>
__device__ void wavefront_dir(const Lattice &L, const float2 *__restrict__ pairs, float *__restrict__ out,
                              Slot *ring, int ring_size, int *cons, float *ll_out, uint32_t *dec = nullptr,
                              int dec_stride = 0) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int Tn = L.Tn, Un = L.Un, st = L.stride;
    const int T1 = Tn - 1, U1 = Un - 1;
    const float2 *pr = pairs + L.base;
    float *o = out + L.base;
    const int cols_per_pass = 32 * nwarps;
    const int ring_used = min(ring_size, Tn);

    for (int col0 = 0; col0 < Un; col0 += cols_per_pass) {
        if (col0 > 0) __syncthreads();  // previous pass complete (its last column is our left boundary)
        // reset ring tags / consumer counters for this pass
        if (Un - col0 > 32) {
            for (int k = threadIdx.x; k < nwarps * ring_used; k += blockDim.x)
                ring[(size_t)(k / ring_used) * ring_size + (k % ring_used)].row = -1;
            if (threadIdx.x < nwarps) cons[threadIdx.x] = 0;
        }
        __syncthreads();

        const int wcol = col0 + 32 * warp;
        if (wcol >= Un) continue;  // warp idle in this pass (still takes part in the barriers above)
        Sweep S;
        S.pr = pr; S.o = o;
        S.Tn = Tn; S.Un = Un; S.st = st; S.T1 = T1; S.U1 = U1;
        S.lane = lane;
        S.j = wcol + lane;
        S.col_ok = S.j < Un;
        const int active = min(32, Un - wcol);
        S.nsteps = Tn + active - 1;
        S.publish = (wcol + 32 < Un) && (warp + 1 < nwarps);   // lane 31's column feeds the next warp
        S.ring_in = ring + (size_t)(warp > 0 ? warp - 1 : 0) * ring_size;
        S.ring_out = ring + (size_t)warp * ring_size;
        S.cons_self = cons + warp;
        S.cons_next = cons + min(warp + 1, nwarps - 1);
        S.ring_mask = ring_size - 1;
        S.backpressure = Tn > ring_size;
        S.override0 = false;
        if constexpr (KIND == kMax) S.dec = dec + (size_t)(wcol / 32) * dec_stride;

        // Exact mode, column 0: the reference builds it with a 32-wide Kogge-Stone scan per tile
        // plus the tile's base value (core.cu:92-110 / :197-215); reproduce that summation order
        // so alpha/beta are bit-identical.  Done up front by warp 0; lane 0 then reads it back.
        const bool col0_scan = (KIND == kExactDense || KIND == kExactCompact) && (wcol == 0);
        if (col0_scan) {
            float base = BETA ? pr[(int64_t)T1 * st + U1].x : 0.0f;
            if (lane == 0) o[BETA ? ((int64_t)T1 * st + U1) : 0] = base;
            for (int p0 = 0; p0 < T1; p0 += 32) {
                const int i = p0 + lane + 1;  // row computed by this lane
                float b = 0.0f;
                if (i <= T1) b = BETA ? pr[(int64_t)(T1 - i) * st + U1].x : pr[(int64_t)(i - 1) * st].x;
#pragma unroll
                for (int k = 1; k < 32; k <<= 1) {
                    const float a = __shfl_up_sync(0xffffffffu, b, k);
                    if (k <= lane) b += a;
                }
                const float v = base + b;
                if (i <= T1) o[BETA ? ((int64_t)(T1 - i) * st + U1) : ((int64_t)i * st)] = v;
                base = __shfl_sync(0xffffffffu, v, 31);
            }
            __syncwarp();
            S.override0 = true;
        }

        float val;
        if (warp > 0) val = sweep_warp<KIND, BETA, kLeftRing, PF>(S);
        else if (col0 > 0 || col0_scan) val = sweep_warp<KIND, BETA, kLeftMem, PF>(S);
        else val = sweep_warp<KIND, BETA, kLeftNone, PF>(S);

        // the thread that owns the last cell reports the log-likelihood seen from this direction
        if (S.j == U1 && ll_out != nullptr) {
            // alpha side: alpha[T-1,U-1] + blank[T-1,U-1] (core.cu:346) ; beta side: beta[0,0]
            *ll_out = BETA ? val : val + pr[(int64_t)T1 * st + U1].x;
        }
    }
}

// grid (2, N) with cluster (2,1,1): rank 0 = alpha, rank 1 = beta (beta_only: grid (1,N), no cluster).
// ws_ll: (2,N) floats {alpha-side ll, beta-side ll}; bad: (N) ints (1 = mismatch guard fired).
template <int KIND, int PF>
__global__ void __launch_bounds__(512, 1) k_wavefront(Problem p, const float2 *__restrict__ pairs,
                                                    float *__restrict__ alphas, float *__restrict__ betas,
                                                    float *__restrict__ ws_ll, int *__restrict__ bad,
                                                    float *__restrict__ costs, int beta_only, int guard, int ring_size,
                                                    GuardPoison poison) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int nwarps = blockDim.x >> 5;
    Slot *ring = reinterpret_cast<Slot *>(smem_raw);
    int *cons = reinterpret_cast<int *>(smem_raw + sizeof(Slot) * (size_t)nwarps * ring_size);
    const int n = blockIdx.y;
    const bool is_beta = beta_only || (blockIdx.x == 1);
    const Lattice L = get_lattice(p, n);
    float *ll = ws_ll + (is_beta ? p.N : 0) + n;
    if (L.ok) {
        if (is_beta) wavefront_dir<KIND, true, PF>(L, pairs, betas, ring, ring_size, cons, ll);
        else wavefront_dir<KIND, false, PF>(L, pairs, alphas, ring, ring_size, cons, ll);
    }
    if (!beta_only) {
        // alpha and beta CTAs of a lattice meet here; release/acquire orders the ll writes.
        __threadfence();
        cluster_arrive_release();
        cluster_wait_acquire();
    } else {
        __syncthreads();
    }
    if (is_beta && threadIdx.x == 0) {
        float cost = NAN;
        int isbad = 0;
        if (L.ok) {
            float b = __ldcg(ws_ll + p.N + n);
            if (lattice_dead(b)) {
                // no alignment of finite log-probability: the reference's class, and no mismatch guard (its ratio
                // is NaN in the reference)
                b = -dead_cost(L.Tn, L.Un, p.compact);
            } else if (!beta_only && guard) {
                // forward/backward mismatch guard, core.cu:346-367
                float a = __ldcg(ws_ll + n);
                if (n == poison.n) a += poison.delta;      // test hook, see rnnt_b200_debug_guard_poison
                const float ratio = fabsf(a - b) / fabsf(fmaxf(a, b));
                if (ratio > 0.001f) {
                    printf("\nWARNING: sample %d [%d, %d] has a forward/backward mismatch %f / %f\n", n, L.Tn,
                           L.Un - 1, a, b);
                    b = (a + b) / 2.0f;
                    isbad = 1;
                }
            }
            cost = -b;
        } else {
            isbad = 1;
        }
        costs[n] = cost;
        if (bad) bad[n] = isbad;
    }
}

// ------------------------------------------------------------------------------------------
// k_align: Viterbi forced alignment of one lattice per CTA, grid (1, N), no cluster.  The alpha wavefront in its
// max-plus form (kMax) writes alpha and one decision word per warp and step; then warp 0 backtracks from
// (Tn-1, Un-1) and writes the frame of every label edge and the best path's score alpha[Tn-1,Un-1] + blank[Tn-1,Un-1].
// dec: (N, ceil(U/32), T+31) words laid out by the bounds T, U (dense: the padded sizes; compact: max_T, max_U); a
// lattice outside them gets score NaN.  frames: dense (N, U-1), compact (sum yn) in the labels' order.
// ------------------------------------------------------------------------------------------
template <int PF>
__global__ void __launch_bounds__(512, 1) k_align(Problem p, const float2 *__restrict__ pairs, float *__restrict__ alphas,
                                                uint32_t *__restrict__ dec, int T, int U, int ring_size,
                                                float *__restrict__ scores, int *__restrict__ frames) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ float s_score;
    const int nwarps = blockDim.x >> 5;
    Slot *ring = reinterpret_cast<Slot *>(smem_raw);
    int *cons = reinterpret_cast<int *>(smem_raw + sizeof(Slot) * (size_t)nwarps * ring_size);
    const int n = blockIdx.y;
    const Lattice L = get_lattice(p, n);
    const bool ok = L.ok && L.Tn <= T && L.Un <= U;
    const int stride = T + 31;
    uint32_t *d = dec + (size_t)n * ((U + 31) / 32) * stride;
    if (threadIdx.x == 0) s_score = NAN;     // ordered before the owner's write by the wavefront's first barrier
    if (ok) wavefront_dir<kMax, false, PF>(L, pairs, alphas, ring, ring_size, cons, &s_score, d, stride);
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    const float score = s_score;
    // no path above -inf (or every path NaN): no alignment, every frame -1
    const bool live = ok && score > -INFINITY;
    int *fr = frames + (p.compact ? L.lab_base : (int64_t)n * (U - 1));
    const int slots = p.compact ? max(L.Un - 1, 0) : U - 1;
    for (int u = (live ? L.Un - 1 : 0) + lane; u < slots; u += 32) fr[u] = -1;
    if (lane == 0) scores[n] = score;
    if (!live) return;
    // Backtrace.  The stored bits already follow the border rules (row 0: 1, column 0: 0), so inside column block w
    // the walk is ul -= bit ul of word s, with s = t + ul falling by one per step (blank: t-1; label: ul-1): one
    // coalesced load brings 32 steps' words (lane k: word s_hi - k) while the block's next 32 are prefetched, every lane
    // walks the 32 steps on shuffled copies (no load on the chain), and lane k keeps its own step's column and bit to
    // write that step's frame afterwards.  A label edge out of ul == 0 enters block w-1 at word t + 31, where the
    // prefetch is dropped; block 0 ends at word 0, cell (0,0).  w, ul and s_hi are warp-uniform.
    int w = (L.Un - 1) >> 5, ul = (L.Un - 1) & 31;
    int s_hi = L.Tn - 1 + ul;
    const uint32_t *blk = d + (size_t)w * stride;
    uint32_t mine = (s_hi - lane >= 0) ? blk[s_hi - lane] : 0u;
    while (true) {
        const int s_next = s_hi - 32;
        const uint32_t next = (s_next - lane >= 0) ? blk[s_next - lane] : 0u;
        int my_ul = 0, my_b = 0;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const uint32_t word = __shfl_sync(0xffffffffu, mine, k);
            const int b = ul >= 0 ? (int)((word >> ul) & 1u) : 0;    // ul == -1: left the block at an earlier step
            if (lane == k) { my_ul = ul; my_b = b; }
            ul -= b;
        }
        if (my_b) fr[32 * w + my_ul - 1] = s_hi - lane - my_ul;       // label edge into column 32w + my_ul at t
        const unsigned out = __ballot_sync(0xffffffffu, my_b && my_ul == 0);
        if (out) {
            s_hi = s_hi - (__ffs(out) - 1) + 31;
            --w;
            ul = 31;
            blk -= stride;
            mine = (s_hi - lane >= 0) ? blk[s_hi - lane] : 0u;
        } else {
            if (s_next < 0) break;
            s_hi = s_next;
            mine = next;
        }
    }
}

// ------------------------------------------------------------------------------------------
// k_grads_pairs: out[cell] = (blank grad, label grad) for every cell of the layout (zeros on
// padding and on the structural zeros).  Elementwise, all SMs.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cell_grads(const Lattice &L, const float2 *__restrict__ pairs,
                                             const float *__restrict__ alphas, const float *__restrict__ betas,
                                             int t, int u, float b00, float lam_scale_dummy, float fastemit_lambda) {
    (void)lam_scale_dummy;
    const int64_t c = L.base + (int64_t)t * L.stride + u;
    const float2 w = pairs[c];
    const float al = alphas[c];
    float gb = 0.0f, gl = 0.0f;
    const bool last_t = (t == L.Tn - 1), last_u = (u == L.Un - 1);
    if (!(last_t && !last_u)) {
        // core.cu:284-294
        float a = al;
        if (!last_t) a += betas[c + L.stride];
        a = expf(a + w.x - b00);
        gb = -a;
    }
    if (!last_u) {
        // core.cu:319-331 ; (1. + lambda) * a is a double multiply in the reference
        float a = al + betas[c + 1];
        a = expf(a + w.y - b00);
        a = (float)((1.0 + (double)fastemit_lambda) * (double)a);
        gl = -a;
    }
    return make_float2(gb, gl);
}

constexpr int kGradThreads = 256;

__global__ void __launch_bounds__(kGradThreads)
k_grads_pairs(Problem p, const float2 *__restrict__ pairs, const float *__restrict__ alphas,
              const float *__restrict__ betas, const int *__restrict__ bad, float fastemit_lambda,
              float2 *__restrict__ out) {
    const int n = blockIdx.y;
    const Lattice L = get_lattice(p, n);
    const int total = p.compact ? (L.ok ? L.Tn * L.Un : 0) : p.T * p.U;  // dense: the whole padded slab
    const int64_t slab = p.compact ? L.base : (int64_t)n * p.T * p.U;
    const int stride = p.compact ? L.stride : p.U;
    const bool live = L.ok && !(bad && bad[n]);
    const float b00 = live ? dead_b00(betas[L.base]) : 0.0f;   // dead lattice: NaN gradients
    for (int r = blockIdx.x * kGradThreads + threadIdx.x; r < total; r += gridDim.x * kGradThreads) {
        const int t = r / stride, u = r - t * stride;
        float2 g = make_float2(0.0f, 0.0f);
        if (live && t < L.Tn && u < L.Un) g = cell_grads(L, pairs, alphas, betas, t, u, b00, 0.0f, fastemit_lambda);
        out[slab + r] = g;
    }
}

// ------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------
cudaError_t launch_prefix(cudaStream_t s, const int *xn, const int *yn, int N, int64_t *mem_pref,
                          int64_t *lab_pref, int *totals) {
    k_prefix<<<1, 1024, 0, s>>>(xn, yn, N, mem_pref, lab_pref, totals);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_gather(cudaStream_t s, const Problem &p, const void *lp, const int *labels, int V, int blank,
                          float2 *pairs, int64_t *loc, int64_t cells_hint, int io_bf16) {
    // cells per lattice: dense T*U; compact unknown on the host -> average * 2, grid-stride covers the rest
    int64_t per = p.compact ? (cells_hint / (p.N > 0 ? p.N : 1)) * 2 + 1 : (int64_t)p.T * p.U;
    int gx = (int)((per + kGatherThreads * kGatherIlp - 1) / (kGatherThreads * kGatherIlp));
    gx = max(1, min(gx, 4096));
    dim3 grid(gx, p.N);
    if (io_bf16) k_gather<__nv_bfloat16><<<grid, kGatherThreads, 0, s>>>(p, static_cast<const __nv_bfloat16 *>(lp), labels, V, blank, pairs, loc);
    else k_gather<float><<<grid, kGatherThreads, 0, s>>>(p, static_cast<const float *>(lp), labels, V, blank, pairs, loc);
    count_launch();
    return cudaGetLastError();
}

// CTA shape of a general wavefront launch over lattices of at most t_hint rows and u_hint columns (0 = unknown)
struct WaveShape {
    int nwarps, ring;
    size_t smem;
};
static WaveShape wave_shape(int t_hint, int u_hint) {
    WaveShape w;
    // warps per CTA: one per 32 lattice columns, at most 16 (more columns -> column passes)
    w.nwarps = (u_hint > 0 ? u_hint + 31 : 512) / 32;
    w.nwarps = max(1, min(w.nwarps, 16));
    // boundary ring: one slot per row when it fits (no back-pressure), else a 128-slot ring
    w.ring = 128;
    if (w.nwarps > 1 && t_hint > 0) {
        while (w.ring < t_hint && (size_t)w.ring * 2 * w.nwarps * sizeof(Slot) <= 160 * 1024) w.ring *= 2;
    }
    w.smem = sizeof(Slot) * (size_t)w.nwarps * w.ring + sizeof(int) * w.nwarps;
    return w;
}

template <int KIND, int PF>
static cudaError_t launch_wavefront_kp(cudaStream_t s, const Problem &p, const float2 *pairs, float *alphas,
                                       float *betas, float *ws_ll, int *bad, float *costs, int beta_only,
                                       int guard, int t_hint, int u_hint) {
    const WaveShape shape = wave_shape(t_hint, u_hint);
    const int nwarps = shape.nwarps, ring = shape.ring;
    const size_t smem = shape.smem;
    static std::atomic<bool> attr_done[kMaxDevices];
    {
        const cudaError_t e = ensure_dyn_smem(k_wavefront<KIND, PF>, attr_done, 200 * 1024);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(beta_only ? 1 : 2, p.N, 1);
    cfg.blockDim = dim3(32 * nwarps, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = beta_only ? 1 : 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    count_launch();
    begin_launch_record(2);
    int32_t *rec = launch_record();
    rec[RNNT_REC_GEN_WARPS] = nwarps; rec[RNNT_REC_GEN_RING] = ring; rec[RNNT_REC_GEN_BETA_ONLY] = beta_only;
    return cudaLaunchKernelEx(&cfg, k_wavefront<KIND, PF>, p, pairs, alphas, betas, ws_ll, bad, costs, beta_only, guard,
                              ring, guard_poison());
}

// The unroll factor of the recurrence loop = its operand prefetch distance.  The exact-LSE body is ~150 instructions
// per step; unrolled 8x, the two instantiations a CTA runs (ring-fed warps + the column-0 warp) are ~40 KB of SASS,
// more than the 32 KB instruction cache behind an SM's schedulers (ncu r1: "no instruction" was the top stall reason).
// At cfg 4 unroll 4 was fastest for the exact flavour and unroll 8 for the fast one.
template <int KIND>
static cudaError_t launch_wavefront_kind(cudaStream_t s, const Problem &p, const float2 *pairs, float *alphas,
                                         float *betas, float *ws_ll, int *bad, float *costs, int beta_only,
                                         int guard, int t_hint, int u_hint) {
    constexpr int PF = (KIND == kFast) ? 8 : 4;
    return launch_wavefront_kp<KIND, PF>(s, p, pairs, alphas, betas, ws_ll, bad, costs, beta_only, guard, t_hint, u_hint);
}

cudaError_t launch_wavefront(cudaStream_t s, bool fast_lse, const Problem &p, const float2 *pairs, float *alphas,
                             float *betas, float *ws_ll, int *bad, float *costs, int beta_only, int t_hint,
                             int u_hint) {
    const int guard = !p.compact;
    switch (lse_kind(fast_lse, p.compact)) {
        case kExactDense:
            return launch_wavefront_kind<kExactDense>(s, p, pairs, alphas, betas, ws_ll, bad, costs, beta_only, guard, t_hint, u_hint);
        case kExactCompact:
            return launch_wavefront_kind<kExactCompact>(s, p, pairs, alphas, betas, ws_ll, bad, costs, beta_only, guard, t_hint, u_hint);
        default:
            return launch_wavefront_kind<kFast>(s, p, pairs, alphas, betas, ws_ll, bad, costs, beta_only, guard, t_hint, u_hint);
    }
}

cudaError_t launch_align(cudaStream_t s, const Problem &p, const float2 *pairs, float *alphas, uint32_t *dec, int T,
                         int U, float *scores, int *frames) {
    // the max-plus step is short like the fast LSE's: the fast flavour's unroll
    constexpr int PF = 8;
    const WaveShape shape = wave_shape(T, U);
    static std::atomic<bool> attr_done[kMaxDevices];
    {
        const cudaError_t e = ensure_dyn_smem(k_align<PF>, attr_done, 200 * 1024);
        if (e != cudaSuccess) return e;
    }
    count_launch();
    begin_launch_record(2);
    int32_t *rec = launch_record();
    rec[RNNT_REC_GEN_WARPS] = shape.nwarps; rec[RNNT_REC_GEN_RING] = shape.ring;
    k_align<PF><<<dim3(1, p.N, 1), 32 * shape.nwarps, shape.smem, s>>>(p, pairs, alphas, dec, T, U, shape.ring, scores,
                                                                       frames);
    return cudaGetLastError();
}

cudaError_t launch_grads_pairs(cudaStream_t s, const Problem &p, const float2 *pairs, const float *alphas,
                               const float *betas, const int *bad, float fastemit_lambda, float2 *out,
                               int64_t cells_hint) {
    int64_t per = p.compact ? (cells_hint / (p.N > 0 ? p.N : 1)) * 2 + 1 : (int64_t)p.T * p.U;
    int gx = (int)((per + kGradThreads - 1) / kGradThreads);
    gx = max(1, min(gx, 8192));
    dim3 grid(gx, p.N);
    k_grads_pairs<<<grid, kGradThreads, 0, s>>>(p, pairs, alphas, betas, bad, fastemit_lambda, out);
    count_launch();
    return cudaGetLastError();
}

}  // namespace rnnt
