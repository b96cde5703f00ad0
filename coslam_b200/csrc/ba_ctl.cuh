// ba_ctl.cuh -- device-side Levenberg-Marquardt control of the submitted bundle adjustment
// (cosl_ba_solver_submit, DESIGN.md section 4).  The host loop of ba.cu (levmar + run_robust) is replayed
// as a state machine: one CUDA graph holds a WHILE node whose body runs one stage per iteration -- a new
// robust round (weights + initial cost), a linearisation, or one LM trial -- selected by IF nodes, then
// ba_ctl_step takes the decision the host takes after reading the scalars back and sets the conditions of
// the next iteration.  Every decision uses the same fp64 operations as the host code, each rounded on its
// own (_rn intrinsics: no FMA contraction), so it takes the same branch for the same scalars.
#pragma once
#include <cuda_runtime.h>

#include "ba_kernels.cuh"

namespace coslam {

enum BaStage { BA_STAGE_ROUND = 0, BA_STAGE_LIN0 = 1, BA_STAGE_LIN = 2, BA_STAGE_TRIAL = 3, BA_NSTAGES = 4 };

// control block (device memory, one per solver)
struct BaCtl {
  double mu, nu, p_eL2, init_eL2, ginf, maxdiag, dp_L2, first_e0;
  int stage;         // the stage the loop body runs in this iteration
  int round, itno, stop, nfev, njev, nlss, totalTrials;
  int statsPending;  // the prep kernel of the next trial computes |g|_inf / max diag (linearisation at itno > 0)
  int ginfPending;   // the eps1 test of this iteration waits for the next trial's scalars
  int copy;          // ba_ctl_accept copies the accepted trial na -> pa, nb -> pb
  int done;
};

// stop reason of a loop ended by cosl_ba_solver_stop
enum { BA_STOP_CALLER = 8 };

// What ba_ctl_step publishes after every decision (cosl_ba_solver_progress).  seq0 is written first and
// seq1 last, each with a fence, so a copy with seq0 != seq1 raced a write.
struct BaProgress {
  unsigned long long seq0, req;  // req: the request the record belongs to
  double p_eL2, init_eL2, mu;
  int round;   // rounds started (the rounds run once the loop has ended)
  int itno;    // counted iterations of the round
  int trials;  // LM trials over all rounds
  int pad;
  unsigned long long seq1;
};

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
  double tau, eps1, eps2, eps3, eps4;
  int rounds, itmax, ns, hasObs, outliers;
  cudaGraphConditionalHandle hLoop, hStage[BA_NSTAGES];
  BaCtlLink* link;
};

__global__ void ba_fill_f64(double* __restrict__ p, long long n, double v) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    p[q] = v;
}

// ---- kernels of an LM trial with mu (and doStats) read from the control block
__global__ void __launch_bounds__(256)
ba_cam_update_ctl(BaDev d, const BaCtl* __restrict__ c, const double* __restrict__ pa, const double* __restrict__ sol,
                  double* __restrict__ dpa, double* __restrict__ na, int addSums, double* __restrict__ zeroBuf,
                  long long zeroCount) {
  ba_cam_update_body(d, pa, sol, dpa, na, c->mu, addSums, zeroBuf, zeroCount);
}

__global__ void __launch_bounds__(256)
ba_back_finish_ctl(BaDev d, const BaCtl* __restrict__ c, const double* __restrict__ pb, double* __restrict__ nb,
                   double* __restrict__ dpb) {
  ba_back_finish_body(d, pb, nb, dpb, c->mu);
}

__global__ void __launch_bounds__(256)
ba_back_cams_points_ctl(BaDev d, const BaCtl* __restrict__ c, const double* __restrict__ pa,
                        const double* __restrict__ sol, double* __restrict__ dpa, double* __restrict__ na, int addSums,
                        int nCamBlocks, double* __restrict__ acc3) {
  ba_back_cams_points_body(d, pa, sol, dpa, na, c->mu, addSums, nCamBlocks, acc3);
}

__global__ void __launch_bounds__(256)
ba_finish_cost_ctl(BaDev d, const BaCtl* __restrict__ c, const double* __restrict__ na, const double* __restrict__ pb,
                   double* __restrict__ nb, const double* __restrict__ acc3, const double* __restrict__ Vinv) {
  ba_finish_cost_body(d, na, pb, nb, acc3, Vinv, c->mu);
}

// ba_prep_kernel with mu and doStats from the control block.  The body is ba_prep_kernel's own: moving
// it into a shared inline function changes the register allocation of ba_prep_kernel.
__global__ void __launch_bounds__(256)
ba_prep_kernel_ctl(BaDev d, const BaCtl* __restrict__ c, int addU, const int* __restrict__ diagBlk,
                   const int* __restrict__ blkCam0, const int* __restrict__ order, int* __restrict__ cnt, int nCnt,
                   int nTiles, double* __restrict__ Vinv, double* __restrict__ zeroBuf, long long zeroCount) {
  const double mu = c->mu;
  const int doStats = c->statsPending;
  for (int q = blockIdx.x * 256 + threadIdx.x; q < nCnt; q += gridDim.x * 256) cnt[q] = 0;
  for (long long q = (long long)blockIdx.x * 256 + threadIdx.x; q < zeroCount; q += (long long)gridDim.x * 256)
    zeroBuf[q] = 0.0;
  if (blockIdx.x == 0 && threadIdx.x < 6) {
    const int slot[6] = {SC_DP_L2, SC_DL, SC_P_L2, SC_FAIL, SC_COST, SC_NONFINITE};
    d.sc[slot[threadIdx.x]] = 0.0;
  }
  if ((int)blockIdx.x < nTiles) {
    ba_tile_init_body(d, mu, addU, diagBlk, blkCam0, order);
    return;
  }
  const long long t = (long long)(blockIdx.x - nTiles) * 256 + threadIdx.x;
  double g = 0, dg = 0;
  if (t < d.n) {
    double I[6] = {0, 0, 0, 0, 0, 0};
    if (t >= d.ncon) {
      const double* V = d.V + 6 * t;
      inv3sym_mu(V, mu, I);
      if (doStats) {
        const double* e = d.eb + 3 * t;
        g = fmax(fabs(e[0]), fmax(fabs(e[1]), fabs(e[2])));
        dg = fmax(V[0], fmax(V[3], V[5]));
      }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) Vinv[6 * t + k] = I[k];
  } else if (doStats && t < (long long)d.n + d.m) {
    const int j = (int)(t - d.n);
    if (j >= d.mcon) {
      const double* U = d.U + 21 * (size_t)j;
      const double* e = d.ea + 6 * (size_t)j;
      dg = fmax(fmax(U[0], U[6]), fmax(fmax(U[11], U[15]), fmax(U[18], U[20])));
#pragma unroll
      for (int k = 0; k < 6; ++k) g = fmax(g, fabs(e[k]));
    }
  }
  if (doStats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      g = fmax(g, __shfl_xor_sync(0xffffffffu, g, o));
      dg = fmax(dg, __shfl_xor_sync(0xffffffffu, dg, o));
    }
    if ((threadIdx.x & 31) == 0) {
      if (g > 0) atomic_max_nonneg(&d.sc[SC_GINF], g);
      if (dg > 0) atomic_max_nonneg(&d.sc[SC_MAXDIAG], dg);
    }
  }
}

// ---- the control kernels (one thread)
// Enter `next`: set the stage conditions and clear the scalars that the stage accumulates into but does
// not clear itself (the host path clears the same slots with memsets).
__device__ void ba_ctl_goto(BaCtl* c, double* sc, const BaCtlParams& P, int next) {
  c->stage = next;
#pragma unroll
  for (int k = 0; k < BA_NSTAGES; ++k) cudaGraphSetConditional(P.hStage[k], k == next ? 1u : 0u);
  if (next == BA_STAGE_ROUND) {
    sc[SC_COST] = 0.0;
    sc[SC_NONFINITE] = 0.0;
  } else if ((next == BA_STAGE_LIN0 || next == BA_STAGE_LIN) && !P.hasObs) {
    sc[SC_GINF] = 0.0;  // otherwise ba_linearize_points clears them
    sc[SC_MAXDIAG] = 0.0;
  } else if (next == BA_STAGE_TRIAL && !P.ns) {  // otherwise the prep kernel clears them
    sc[SC_DP_L2] = sc[SC_DL] = sc[SC_P_L2] = sc[SC_FAIL] = sc[SC_COST] = sc[SC_NONFINITE] = 0.0;
  }
}

// Has the caller asked to stop this request?  Read at every transition into a further stage: LIN after a
// finished iteration, TRIAL after a linearisation or a rejected trial, ROUND for the next round.  The stop
// word is written by a copy on another stream while the loop runs, hence the volatile load.
__device__ bool ba_ctl_stop_asked(const BaCtlParams& P) {
  const volatile unsigned long long* w = &P.link->req;
  return w[1] == w[0];
}

// end of a robust round (after levmar returned): run_robust's bookkeeping, then the next round or the end
__device__ void ba_ctl_end_round(BaCtl* c, double* sc, const BaCtlParams& P) {
  if (c->itno >= P.itmax && !c->stop) c->stop = 3;
  if (c->first_e0 < 0) c->first_e0 = c->init_eL2;
  c->totalTrials += c->nlss;
  if (++c->round < P.rounds && c->stop != BA_STOP_CALLER) {
    if (!ba_ctl_stop_asked(P)) {
      ba_ctl_goto(c, sc, P, BA_STAGE_ROUND);
      return;
    }
    c->stop = BA_STOP_CALLER;  // no further round: the round that ended reports the stop
  }
  c->done = 1;
  c->stage = -1;
#pragma unroll
  for (int k = 0; k < BA_NSTAGES; ++k) cudaGraphSetConditional(P.hStage[k], 0u);
  cudaGraphSetConditional(P.hLoop, 0u);
  sc[SC_COST] = 0.0;  // the outlier count of the pass after the loop
}

// end of an LM iteration (the inner loop of levmar has broken out)
__device__ void ba_ctl_end_iter(BaCtl* c, double* sc, const BaCtlParams& P) {
  if (c->p_eL2 <= P.eps3) c->stop = 3;
  ++c->itno;
  if (c->itno < P.itmax && !c->stop && ba_ctl_stop_asked(P)) c->stop = BA_STOP_CALLER;
  if (c->itno < P.itmax && !c->stop)
    ba_ctl_goto(c, sc, P, BA_STAGE_LIN);
  else
    ba_ctl_end_round(c, sc, P);
}

// Into TRIAL after a linearisation or a rejected trial, unless the caller asked to stop: then the round
// ends without counting the unfinished iteration (as the late eps1 test does).
__device__ void ba_ctl_to_trial(BaCtl* c, double* sc, const BaCtlParams& P) {
  if (ba_ctl_stop_asked(P)) {
    c->stop = BA_STOP_CALLER;
    ba_ctl_end_round(c, sc, P);
  } else {
    ba_ctl_goto(c, sc, P, BA_STAGE_TRIAL);
  }
}

// the progress record of the decision just taken
__device__ void ba_ctl_publish(const BaCtl* c, BaCtlLink* L) {
  volatile BaProgress* g = &L->prog;
  const unsigned long long k = g->seq1 + 1;
  g->seq0 = k;
  __threadfence();
  g->req = L->req;
  g->round = c->done ? c->round : c->round + 1;
  g->itno = c->itno;
  // end_round has added the round's trials; the ROUND stage clears nlss
  g->trials = c->totalTrials + ((c->done || c->stage == BA_STAGE_ROUND) ? 0 : c->nlss);
  g->p_eL2 = c->p_eL2;
  g->init_eL2 = c->init_eL2;
  g->mu = c->mu;
  __threadfence();
  g->seq1 = k;
}

__global__ void ba_ctl_init(BaCtl* __restrict__ c, double* __restrict__ sc) {
  if (threadIdx.x != 0) return;
  c->mu = c->nu = c->p_eL2 = c->init_eL2 = c->ginf = c->maxdiag = c->dp_L2 = 0.0;
  c->first_e0 = -1.0;
  c->stage = BA_STAGE_ROUND;  // the defaults of the graph's conditions: loop on, ROUND on
  c->round = c->itno = c->stop = c->nfev = c->njev = c->nlss = c->totalTrials = 0;
  c->statsPending = c->ginfPending = c->copy = c->done = 0;
  sc[SC_COST] = 0.0;
  sc[SC_NONFINITE] = 0.0;
}

__device__ void ba_ctl_decide(BaCtl* __restrict__ c, double* __restrict__ sc, const BaCtlParams& P) {
  const double EPS_SQ = 1e-24;
  c->copy = 0;
  switch (c->stage) {
    case BA_STAGE_ROUND: {  // levmar's initial cost
      c->nfev = 1;
      c->njev = c->nlss = 0;
      c->mu = 0.0;
      c->nu = 2.0;
      c->stop = 0;
      c->itno = 0;
      c->statsPending = c->ginfPending = 0;
      const double p = sc[SC_COST];
      c->p_eL2 = c->init_eL2 = p;
      c->ginf = c->maxdiag = c->dp_L2 = 0.0;
      if (!(isfinite(p) && sc[SC_NONFINITE] == 0.0)) c->stop = 7;
      if (!c->stop && c->itno < P.itmax)
        ba_ctl_goto(c, sc, P, BA_STAGE_LIN0);
      else
        ba_ctl_end_round(c, sc, P);
      return;
    }
    case BA_STAGE_LIN0:
    case BA_STAGE_LIN: {
      ++c->njev;
      c->statsPending = (c->itno > 0 && P.ns) ? 1 : 0;
      if (c->itno == 0) {
        c->ginfPending = 0;
        c->ginf = sc[SC_GINF];
        c->maxdiag = sc[SC_MAXDIAG];
        if (c->ginf <= P.eps1) {
          c->stop = 1;
          ba_ctl_end_round(c, sc, P);  // the for loop is left before its increment: itno stays 0
          return;
        }
        c->mu = __dmul_rn(P.tau, c->maxdiag);
      } else {
        c->ginfPending = 1;
      }
      ba_ctl_to_trial(c, sc, P);
      return;
    }
    case BA_STAGE_TRIAL: {
      ++c->nlss;
      ++c->nfev;
      c->statsPending = 0;
      if (c->ginfPending) {
        c->ginfPending = 0;
        c->ginf = sc[SC_GINF];
        c->maxdiag = sc[SC_MAXDIAG];
        if (c->ginf <= P.eps1) {  // the eps1 test of this iteration: the trial just run never happened
          --c->nlss;
          --c->nfev;
          c->stop = 1;
          ba_ctl_end_round(c, sc, P);
          return;
        }
      }
      if (sc[SC_FAIL] == 0.0) {
        const double dp_L2 = sc[SC_DP_L2], dL = sc[SC_DL], p_L2 = sc[SC_P_L2];
        c->dp_L2 = dp_L2;
        if (dp_L2 <= __dmul_rn(__dmul_rn(P.eps2, P.eps2), p_L2)) {
          c->stop = 2;
          ba_ctl_end_iter(c, sc, P);
          return;
        }
        if (dp_L2 >= __ddiv_rn(__dadd_rn(p_L2, P.eps2), EPS_SQ)) {
          c->stop = 4;
          ba_ctl_end_iter(c, sc, P);
          return;
        }
        const double pdp_eL2 = sc[SC_COST];
        if (!isfinite(pdp_eL2) || sc[SC_NONFINITE] != 0.0) {
          c->stop = 7;
          ba_ctl_end_iter(c, sc, P);
          return;
        }
        const double p_eL2 = c->p_eL2;
        const double dF = __dadd_rn(p_eL2, -pdp_eL2);
        if (dF > 0 && dL > 0) {
          double tmp = __dadd_rn(__ddiv_rn(__dmul_rn(2.0, dF), dL), -1.0);
          tmp = __dadd_rn(1.0, -__dmul_rn(__dmul_rn(tmp, tmp), tmp));
          const double third = 1.0 / 3.0;
          c->mu = __dmul_rn(c->mu, tmp < third ? third : tmp);  // std::max(tmp, 1/3): NaN stays NaN
          c->nu = 2.0;
          const double sp = __dsqrt_rn(p_eL2);
          if (__dadd_rn(sp, -__dsqrt_rn(pdp_eL2)) < __dmul_rn(P.eps4, sp)) c->stop = 6;
          c->copy = 1;
          c->p_eL2 = pdp_eL2;
          ba_ctl_end_iter(c, sc, P);
          return;
        }
      }
      c->mu = __dmul_rn(c->mu, c->nu);
      const double nu2 = __dmul_rn(c->nu, 2.0);
      if (!(nu2 > c->nu) || !isfinite(c->mu)) {
        c->stop = 5;
        ba_ctl_end_iter(c, sc, P);
        return;
      }
      c->nu = nu2;
      ba_ctl_to_trial(c, sc, P);
      return;
    }
    default:
      return;
  }
}

__global__ void ba_ctl_step(BaCtl* __restrict__ c, double* __restrict__ sc, BaCtlParams P) {
  if (threadIdx.x != 0) return;
  ba_ctl_decide(c, sc, P);
  ba_ctl_publish(c, P.link);
}

// accepted trial: pa <- na, pb <- nb (the host path swaps the pointers instead; the graph keeps its own)
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
