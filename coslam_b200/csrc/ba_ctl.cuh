// ba_ctl.cuh -- the device driver of the LM control (ba_lm.cuh) for the submitted bundle adjustment
// (cosl_ba_solver_submit, DESIGN.md section 4.5).  One CUDA graph holds a WHILE node whose body runs one stage
// per iteration, selected by IF nodes; then ba_ctl_step takes the decision that the host driver takes after
// reading the scalars back, and sets the conditions of the next iteration.
#pragma once
#include <cuda_runtime.h>

#include "ba_lm.cuh"

namespace coslam {

// Device memory shared by the solver's stream and the side stream of stop / progress (one per solver):
// req is the number of the submitted request, written on the solver's stream before its graph; stop is
// the number of the request the caller asked to stop, written on the side stream.  They match only while
// the request that was asked to stop runs.
struct BaCtlLink {
  unsigned long long req, stop;
  BaProgress prog;
};

// fixed for the life of a graph (the options of a solver do not change)
struct BaCtlParams {
  BaLmParams lm;
  cudaGraphConditionalHandle hLoop, hStage[BA_NSTAGES];
  BaCtlLink* link;
};

__global__ void ba_fill_f64(double* __restrict__ p, long long n, double v) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    p[q] = v;
}

__device__ void ba_ctl_clear(double* sc, unsigned mask) {
#pragma unroll
  for (int k = 0; k < SC_NTOT; ++k)
    if (mask >> k & 1u) sc[k] = 0.0;
}

__global__ void ba_ctl_init(BaCtl* __restrict__ c, double* __restrict__ sc, BaLmParams P) {
  if (threadIdx.x != 0) return;
  ba_lm_start(*c);  // the defaults of the graph's conditions: loop on, ROUND on
  ba_ctl_clear(sc, ba_lm_cleared(*c, P));
}

// One decision (one thread): clear what the next stage needs cleared, set the conditions of the next iteration
// and publish the progress record.  The stop word is written by a copy on another stream while the loop runs,
// hence the volatile load.
__global__ void ba_ctl_step(BaCtl* __restrict__ c, double* __restrict__ sc, BaCtlParams P) {
  if (threadIdx.x != 0) return;
  const volatile unsigned long long* w = &P.link->req;
  ba_lm_decide(*c, sc, P.lm, w[1] == w[0]);
  ba_ctl_clear(sc, ba_lm_cleared(*c, P.lm));
#pragma unroll
  for (int k = 0; k < BA_NSTAGES; ++k) cudaGraphSetConditional(P.hStage[k], k == c->stage ? 1u : 0u);
  if (c->done) cudaGraphSetConditional(P.hLoop, 0u);
  volatile BaProgress* g = &P.link->prog;
  const unsigned long long k = g->seq1 + 1;
  g->seq0 = k;
  __threadfence();
  g->req = P.link->req;
  ba_lm_progress(*c, *g);
  __threadfence();
  g->seq1 = k;
}

// accepted trial: pa <- na, pb <- nb (the host driver swaps the pointers instead; the graph keeps its own)
__global__ void __launch_bounds__(256)
ba_ctl_accept(const BaCtl* __restrict__ c, double* __restrict__ pa, const double* __restrict__ na, long long nA,
              double* __restrict__ pb, const double* __restrict__ nb, long long nB) {
  if (!c->copy) return;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nA + nB; q += stride) {
    if (q < nA)
      pa[q] = na[q];
    else
      pb[q - nA] = nb[q - nA];
  }
}

}  // namespace coslam
