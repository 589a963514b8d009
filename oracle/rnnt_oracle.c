/*
 * oracle/rnnt_oracle.c -- CPU restatement of the RNN-Transducer loss + gradient of
 * 1ytic/warp-rnnt.  TEST INFRASTRUCTURE ONLY: this file is the checker, never the product.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load it.  The product path (warp_rnnt_b200) never links or calls anything in oracle/.
 *
 * What it restates (all citations are the reference's <file>:<line>):
 *   alpha recurrence      core.cu:41-141   (row 0 :80-90, column 0 :92-110, interior :112-134)
 *   beta recurrence       core.cu:143-246  (corner :171-173, last row :185-195, last col :197-215,
 *                                           interior :217-239)
 *   log_sum_exp           core.cu:26-39    max + log1p(exp(-|a-b|))
 *   blank gradients       core.cu:260-295
 *   label gradients       core.cu:297-332  (FastEmit factor (1+lambda) on label grads only :327-329)
 *   costs + mismatch guard core.cu:334-370
 *   gathered (V=2) form   core_gather.cu:37-357  (same algorithm, blank->column 0, label->column 1)
 *   compact gather        core_compact.cu:403-436 (loc = label id, blank on the last column)
 *   compact core          core_compact.cu:29-358  (ragged offsets memPref[n] + t*Un + u)
 *   compact scatter       core_compact.cu:456-484 (x grad_cost[n]; label written only if loc != blank)
 *
 * The reference has no CPU implementation; the per-sample double loop is the awni
 * ref_transduce.py style the reference README names as the algorithm's origin (README.md:6,11).
 * Pinned against the golden vectors of pytorch_binding/warp_rnnt/test.py (tests/golden/) and,
 * on the GPU, against the recorded outputs of the compiled unmodified reference (tests/golden/).
 *
 * Two arithmetic flavours are generated from one body: f64 (truth) and f32 (same operation
 * order as the reference kernels, CPU libm expf/log1pf -- close to, not bit-equal with, CUDA's).
 *
 * Lattices are independent (core.cu:49 batch on blockIdx.z) -> OpenMP over n when built -fopenmp.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

int rnnt_oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void rnnt_oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ------------------------------------------------------------------ f64 flavour */
#define REAL double
#define SUFFIX(name) name##_f64
#define R_EXP exp
#define R_LOG1P log1p
#define R_FABS fabs
#define R_FMAX fmax
#include "rnnt_oracle_body.inc"
#undef REAL
#undef SUFFIX
#undef R_EXP
#undef R_LOG1P
#undef R_FABS
#undef R_FMAX

/* ------------------------------------------------------------------ f32 flavour */
#define REAL float
#define SUFFIX(name) name##_f32
#define R_EXP expf
#define R_LOG1P log1pf
#define R_FABS fabsf
#define R_FMAX fmaxf
#include "rnnt_oracle_body.inc"
#undef REAL
#undef SUFFIX
#undef R_EXP
#undef R_LOG1P
#undef R_FABS
#undef R_FMAX
