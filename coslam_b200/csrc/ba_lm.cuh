// ba_lm.cuh -- the Levenberg-Marquardt control of the bundle adjustment (DESIGN.md 4.1, 4.5): one decision
// function, stepped after every stage of the robust loop by two drivers -- the host loop of cosl_ba_solver_run
// (ba.cu, run_host) and the one-thread ba_ctl_step of the submitted graph (ba_ctl.cuh).  The loop runs one
// stage at a time -- a new robust round (weights + initial cost), a linearisation, or one LM trial -- and the
// decision reads that stage's scalars and picks the next one.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

namespace coslam {

// the scalar slots the stages accumulate into (device memory, read back by the host driver)
enum BaScalar {
  SC_COST = 0,     // sum w |e|^2 of the evaluated parameter set
  SC_DP_L2 = 1,    // |dp|^2
  SC_DL = 2,       // dp . (mu dp + g)
  SC_P_L2 = 3,     // |p|^2 over free parameters
  SC_NONFINITE = 4,
  SC_NSUM = 8,     // [0, SC_NSUM) are sums (all-reduce sum)
  SC_GINF = 8,     // |g|_inf                 (all-reduce max)
  SC_MAXDIAG = 9,  // max diag(U, V)
  SC_FAIL = 10,    // Cholesky break-down flag
  SC_NTOT = 16
};

enum BaStage { BA_STAGE_ROUND = 0, BA_STAGE_LIN0 = 1, BA_STAGE_LIN = 2, BA_STAGE_TRIAL = 3, BA_NSTAGES = 4 };

// stop reason of a loop ended by cosl_ba_solver_stop
enum { BA_STOP_CALLER = 8 };

// the state of the loop (host memory for run, device memory for submit)
struct BaCtl {
  double mu, nu, p_eL2, init_eL2, ginf, maxdiag, dp_L2, first_e0;
  int stage;         // the stage the loop runs next
  int round, itno, stop, nfev, njev, nlss, totalTrials;
  int statsPending;  // the stage that runs next computes |g|_inf / max diag for the eps1 test (at itno > 0 a
                     // linearisation with free cameras leaves them to the prep kernel of the next trial)
  int ginfPending;   // the eps1 test of this iteration waits for the next trial's scalars
  int copy;          // the trial just decided was accepted: na -> pa, nb -> pb
  int rated;         // the trial just decided reached the gain-ratio test (what verbose prints)
  int done;
};

// fixed for the life of a loop
struct BaLmParams {
  double tau, eps1, eps2, eps3, eps4;
  int rounds, itmax, ns, hasObs, outliers;
  int fixedTrials;  // > 0: cosl_ba_solver_run_fixed -- no eps1..eps4 stops, stop 3 after that many trials
};

// What a driver publishes after every decision (cosl_ba_solver_progress).  seq0 is written first and seq1
// last, so a copy with seq0 != seq1 raced a write.
struct BaProgress {
  unsigned long long seq0, req;  // req: the request the record belongs to
  double p_eL2, init_eL2, mu;
  int round;   // rounds started (the rounds run once the loop has ended)
  int itno;    // counted iterations of the round
  int trials;  // LM trials over all rounds
  int pad;
  unsigned long long seq1;
};

// The decisions round every fp64 operation on its own, so that the device (where nvcc would contract
// a * b + c into an FMA) takes the host's branch for the same scalars; the host build does not contract.
__host__ __device__ inline double lm_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline double lm_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double lm_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ inline double lm_sqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
__host__ __device__ inline bool lm_finite(double a) {
#ifdef __CUDA_ARCH__
  return isfinite(a);
#else
  return std::isfinite(a);
#endif
}

__host__ __device__ inline void ba_lm_start(BaCtl& c) {
  c.mu = c.nu = c.p_eL2 = c.init_eL2 = c.ginf = c.maxdiag = c.dp_L2 = 0.0;
  c.first_e0 = -1.0;
  c.stage = BA_STAGE_ROUND;
  c.round = c.itno = c.stop = c.nfev = c.njev = c.nlss = c.totalTrials = 0;
  c.statsPending = c.ginfPending = c.copy = c.rated = c.done = 0;
}

// The scalar slots that the next stage accumulates into but does not clear itself (bit k: sc[k]).  After the
// loop: the outlier count of the pass that follows it.
__host__ __device__ inline unsigned ba_lm_cleared(const BaCtl& c, const BaLmParams& P) {
  if (c.done) return P.outliers ? 1u << SC_COST : 0u;
  switch (c.stage) {
    case BA_STAGE_ROUND:
      return 1u << SC_COST | 1u << SC_NONFINITE;
    case BA_STAGE_LIN0:
    case BA_STAGE_LIN:  // with observations ba_linearize_points clears them
      return P.hasObs ? 0u : 1u << SC_GINF | 1u << SC_MAXDIAG;
    case BA_STAGE_TRIAL:  // with free cameras the prep kernel clears them
      return P.ns ? 0u
                  : 1u << SC_DP_L2 | 1u << SC_DL | 1u << SC_P_L2 | 1u << SC_FAIL | 1u << SC_COST |
                        1u << SC_NONFINITE;
    default:
      return 0u;
  }
}

// the fields of the progress record after a decision
__host__ __device__ inline void ba_lm_progress(const BaCtl& c, volatile BaProgress& g) {
  g.round = c.done ? c.round : c.round + 1;
  g.itno = c.itno;
  g.trials = c.totalTrials + ((c.done || c.stage == BA_STAGE_ROUND) ? 0 : c.nlss);  // the round's trials are added
  g.p_eL2 = c.p_eL2;                                                                // when it ends
  g.init_eL2 = c.init_eL2;
  g.mu = c.mu;
}

// end of a robust round: the next round, or the end of the loop
__host__ __device__ inline void ba_lm_end_round(BaCtl& c, const BaLmParams& P, bool stopAsked) {
  if (c.itno >= P.itmax && !c.stop) c.stop = 3;
  if (c.first_e0 < 0) c.first_e0 = c.init_eL2;
  c.totalTrials += c.nlss;
  if (++c.round < P.rounds && c.stop != BA_STOP_CALLER) {
    if (!stopAsked) {
      c.stage = BA_STAGE_ROUND;
      return;
    }
    c.stop = BA_STOP_CALLER;  // no further round: the round that ended reports the stop
  }
  c.done = 1;
  c.stage = -1;
}

// end of an LM iteration: the next linearisation, unless the round ends
__host__ __device__ inline void ba_lm_end_iter(BaCtl& c, const BaLmParams& P, bool stopAsked) {
  if (!P.fixedTrials && c.p_eL2 <= P.eps3) c.stop = 3;
  ++c.itno;
  if (c.itno < P.itmax && !c.stop && stopAsked) c.stop = BA_STOP_CALLER;
  if (c.itno < P.itmax && !c.stop) {
    c.stage = BA_STAGE_LIN;
    c.statsPending = !P.fixedTrials;
  } else {
    ba_lm_end_round(c, P, stopAsked);
  }
}

// Into a trial after a linearisation or a rejected trial, unless the caller asked to stop: then the round
// ends without counting the unfinished iteration (as the late eps1 test does).
__host__ __device__ inline void ba_lm_to_trial(BaCtl& c, const BaLmParams& P, bool stopAsked) {
  if (stopAsked) {
    c.stop = BA_STOP_CALLER;
    ba_lm_end_round(c, P, stopAsked);
  } else {
    c.stage = BA_STAGE_TRIAL;
  }
}

// The decision after the stage c.stage has run, from its scalars sc: control flow identical to
// oracle/ba_oracle.cpp:levmar and run_robust.  After the first iteration the eps1 test is evaluated one stage
// late: the statistics of a linearisation arrive with the scalars of the next trial, which is discarded if
// the test fires -- it only wrote the trial buffers.  stopAsked: the caller asked to stop this request (read
// once per decision); the checks sit at every transition into a further stage -- LIN after a finished
// iteration, TRIAL after a linearisation or a rejected trial, ROUND for the next round.
__host__ __device__ inline void ba_lm_decide(BaCtl& c, const double* sc, const BaLmParams& P, bool stopAsked) {
  const double EPS_SQ = 1e-24;
  c.copy = c.rated = 0;
  switch (c.stage) {
    case BA_STAGE_ROUND: {  // the initial cost of the round
      c.nfev = 1;
      c.njev = c.nlss = 0;
      c.mu = 0.0;
      c.nu = 2.0;
      c.stop = 0;
      c.itno = 0;
      c.statsPending = c.ginfPending = 0;
      const double p = sc[SC_COST];
      c.p_eL2 = c.init_eL2 = p;
      c.ginf = c.maxdiag = c.dp_L2 = 0.0;
      if (!(lm_finite(p) && sc[SC_NONFINITE] == 0.0)) c.stop = 7;
      if (!c.stop && c.itno < P.itmax)
        c.stage = BA_STAGE_LIN0;
      else
        ba_lm_end_round(c, P, stopAsked);
      return;
    }
    case BA_STAGE_LIN0:
    case BA_STAGE_LIN: {
      ++c.njev;
      c.statsPending = c.itno > 0 && P.ns && !P.fixedTrials;
      if (c.itno == 0) {
        c.ginfPending = 0;
        c.ginf = sc[SC_GINF];
        c.maxdiag = sc[SC_MAXDIAG];
        if (!P.fixedTrials && c.ginf <= P.eps1) {
          c.stop = 1;
          ba_lm_end_round(c, P, stopAsked);  // the iteration is left before it is counted: itno stays 0
          return;
        }
        c.mu = lm_mul(P.tau, c.maxdiag);
      } else {
        c.ginfPending = !P.fixedTrials;
      }
      ba_lm_to_trial(c, P, stopAsked);
      return;
    }
    case BA_STAGE_TRIAL: {
      ++c.nlss;
      ++c.nfev;
      c.statsPending = 0;
      if (c.ginfPending) {
        c.ginfPending = 0;
        c.ginf = sc[SC_GINF];
        c.maxdiag = sc[SC_MAXDIAG];
        if (c.ginf <= P.eps1) {  // the eps1 test of this iteration: the trial just run never happened
          --c.nlss;
          --c.nfev;
          c.stop = 1;
          ba_lm_end_round(c, P, stopAsked);
          return;
        }
      }
      if (sc[SC_FAIL] == 0.0) {
        const double dp_L2 = sc[SC_DP_L2], dL = sc[SC_DL], p_L2 = sc[SC_P_L2];
        c.dp_L2 = dp_L2;
        if (!P.fixedTrials && dp_L2 <= lm_mul(lm_mul(P.eps2, P.eps2), p_L2)) {
          c.stop = 2;
          ba_lm_end_iter(c, P, stopAsked);
          return;
        }
        if (!P.fixedTrials && dp_L2 >= lm_div(lm_add(p_L2, P.eps2), EPS_SQ)) {
          c.stop = 4;
          ba_lm_end_iter(c, P, stopAsked);
          return;
        }
        const double pdp_eL2 = sc[SC_COST];
        if (!lm_finite(pdp_eL2) || sc[SC_NONFINITE] != 0.0) {
          c.stop = 7;
          ba_lm_end_iter(c, P, stopAsked);
          return;
        }
        c.rated = 1;
        const double p_eL2 = c.p_eL2;
        const double dF = lm_add(p_eL2, -pdp_eL2);
        if (dF > 0 && dL > 0) {
          double tmp = lm_add(lm_div(lm_mul(2.0, dF), dL), -1.0);
          tmp = lm_add(1.0, -lm_mul(lm_mul(tmp, tmp), tmp));
          const double third = 1.0 / 3.0;
          c.mu = lm_mul(c.mu, tmp < third ? third : tmp);  // std::max(tmp, 1/3): NaN stays NaN
          c.nu = 2.0;
          const double sp = lm_sqrt(p_eL2);
          if (!P.fixedTrials && lm_add(sp, -lm_sqrt(pdp_eL2)) < lm_mul(P.eps4, sp)) c.stop = 6;
          c.copy = 1;
          c.p_eL2 = pdp_eL2;
        }
      }
      if (P.fixedTrials && c.nlss >= P.fixedTrials) c.stop = 3;
      if (c.copy || c.stop) {
        ba_lm_end_iter(c, P, stopAsked);
        return;
      }
      c.mu = lm_mul(c.mu, c.nu);
      const double nu2 = lm_mul(c.nu, 2.0);
      if (!(nu2 > c.nu) || !lm_finite(c.mu)) {
        c.stop = 5;
        ba_lm_end_iter(c, P, stopAsked);
        return;
      }
      c.nu = nu2;
      ba_lm_to_trial(c, P, stopAsked);
      return;
    }
    default:
      return;
  }
}

}  // namespace coslam
