/*
 * softmin.h — the softmin weight every partial record of the reduction is built and merged with: K1's three epilogues
 * (rollout_kernel.cuh, rollout_kernel_ar_ws.cuh, rollout_kernel_nn_tc.cuh), K2 and KX (combine_kernel.cuh), and the host
 * twin of the merge (host_twins.cpp: mppib_host_merge_records). One definition, so that they cannot drift.
 */
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define MPPIB_SOFTMIN_FN __host__ __device__ __forceinline__
#else
#define MPPIB_SOFTMIN_FN inline
#endif

namespace mppib
{
// w = expf(-(c - beta) / lambda) (normExpTransform, mppi_common.cu:958-966) of a cost c against a baseline beta <= c, and
// exactly 0 for c = +inf. With a finite baseline expf(-inf) is 0 already, so this changes one case only: a partial whose
// every cost is +inf (a block of samples an out-of-tree cost marks infeasible, or whose cost overflowed) has baseline +inf,
// and expf(-(inf - inf)) would be NaN — which no later rescale removes (0 * NaN = NaN), so U, the normaliser and sum w^2
// would all come out NaN while the reference, with its one global baseline, weights those samples 0. Here such a partial
// is empty (eta = sum w^2 = V = 0), a merge of empty records is empty, and with every cost +inf U = 0 / 0 = NaN as in the
// reference. A NaN cost still gives a NaN weight.
MPPIB_SOFTMIN_FN float softmin_weight(float c, float beta, float lambda_inv)
{
  return c == INFINITY ? 0.0f : expf(-lambda_inv * (c - beta));
}
}  // namespace mppib
