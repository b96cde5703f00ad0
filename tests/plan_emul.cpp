// plan_emul.cpp -- CPU check of coslam_b200/csrc/ba_plan.h (test infrastructure).
// Builds a random SPD reduced camera system with a given co-visibility pattern, executes the task
// list of the plan SEQUENTIALLY in ticket order with plain loops -- asserting that every wait
// condition of a task already holds when its turn comes (the list is a topological order, which is
// what makes the spinning ticket scheduler on the device deadlock-free) -- and compares the
// solution with a dense Cholesky solve.
//   usage: plan_emul <mf> <pattern: band|dense|random> <param> [ndDepth]
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../coslam_b200/csrc/ba_plan.h"

using namespace coslam;

static double* tile(std::vector<double>& S, int idx) { return &S[(size_t)idx * BA_TILE]; }

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const int mf = std::atoi(argv[1]);
  const std::string pat = argv[2];
  const double param = std::atof(argv[3]);
  const int depth = argc > 4 ? std::atoi(argv[4]) : -1;
  std::mt19937_64 rng(1234 + mf);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::vector<uint8_t> adj((size_t)mf * mf, 0);
  for (int a = 0; a < mf; ++a)
    for (int b = a; b < mf; ++b) {
      bool on = (a == b);
      if (pat == "band") on = on || (b - a) <= (int)param;
      if (pat == "dense") on = true;
      if (pat == "random") on = on || (std::abs(U(rng)) < param) || (b - a) <= 2;
      adj[(size_t)a * mf + b] = adj[(size_t)b * mf + a] = on ? 1 : 0;
    }
  const int ns = 6 * mf;
  // dense SPD matrix with that block pattern: strictly diagonally dominant
  std::vector<double> A((size_t)ns * ns, 0.0), rhs(ns);
  for (int a = 0; a < mf; ++a)
    for (int b = a; b < mf; ++b)
      if (adj[(size_t)a * mf + b])
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) {
            if (a == b && c < r) continue;
            const double v = U(rng);
            A[(size_t)(6 * a + r) * ns + 6 * b + c] = v;
            A[(size_t)(6 * b + c) * ns + 6 * a + r] = v;
          }
  for (int i = 0; i < ns; ++i) {
    double s = 0;
    for (int j = 0; j < ns; ++j)
      if (j != i) s += std::fabs(A[(size_t)i * ns + j]);
    A[(size_t)i * ns + i] = s + 1.0 + std::fabs(U(rng));
    rhs[i] = U(rng);
  }
  BaPlan P = ba_make_plan(mf, adj, depth);
  const int nb = P.nb;
  // scatter into tiles (lower triangle in the PERMUTED order)
  const int ntAll = P.nTiles + P.nScratch;
  // scratch tiles start with garbage: the first update must overwrite them
  std::vector<double> S((size_t)ntAll * BA_TILE, 0.0), b((size_t)nb * BA_TB, 0.0), bS((size_t)std::max(1, P.nScratch) * BA_TB, 777.0);
  for (size_t e = (size_t)P.nTiles * BA_TILE; e < S.size(); ++e) S[e] = 1e300;
  for (int a = 0; a < mf; ++a)
    for (int c = 0; c < mf; ++c) {
      if (!adj[(size_t)a * mf + c]) continue;
      for (int r = 0; r < 6; ++r)
        for (int q = 0; q < 6; ++q) {
          const int bi = P.camBlk[a], bj = P.camBlk[c];
          const int ri = P.camOff[a] + r, rj = P.camOff[c] + q;
          if (bi < bj || (bi == bj && ri < rj)) continue;  // keep row >= col
          const int t = P.tileIdx[(size_t)bi * nb + bj];
          if (t < 0 || t >= P.nTilesOrig) {
            std::printf("FAIL: structural tile missing (%d,%d)\n", bi, bj);
            return 1;
          }
          tile(S, t)[rj * BA_TB + ri] = A[(size_t)(6 * a + r) * ns + 6 * c + q];
        }
    }
  for (int a = 0; a < mf; ++a)
    for (int r = 0; r < 6; ++r) b[(size_t)P.camBlk[a] * BA_TB + P.camOff[a] + r] = rhs[6 * a + r];
  // sequential execution in ticket order
  std::vector<int> cnt(P.nCounters, 0);
  std::vector<double> Linv((size_t)nb * BA_TILE, 0.0), y((size_t)nb * BA_TB, 0.0), x((size_t)nb * BA_TB, 0.0);
  for (size_t ti = 0; ti < P.tasks.size(); ++ti) {
    const BaTask& t = P.tasks[ti];
    const int wi[3] = {t.w0i, t.w1i, t.w2i}, wv[3] = {t.w0v, t.w1v, t.w2v};
    for (int w = 0; w < 3; ++w)
      if (wi[w] >= 0 && cnt[wi[w]] < wv[w]) {
        std::printf("FAIL: task %zu (type %d k %d i %d) not ready: cnt[%d]=%d < %d\n", ti, t.type, t.k, t.i,
                    wi[w], cnt[wi[w]], wv[w]);
        return 1;
      }
    if (t.type == BA_T_UPD && cnt[t.w0i] != t.w0v) {
      std::printf("FAIL: update out of sequence\n");
      return 1;
    }
    const int bk = P.blkRows[t.k];
    if (t.type == BA_T_POTRF) {
      double* C = tile(S, t.tC);
      for (int k = 0; k < bk; ++k) {
        double d = C[k * BA_TB + k];
        if (!(d > 0)) {
          std::printf("FAIL: non-positive pivot\n");
          return 1;
        }
        d = std::sqrt(d);
        C[k * BA_TB + k] = d;
        for (int i = k + 1; i < bk; ++i) C[k * BA_TB + i] /= d;
        for (int j = k + 1; j < bk; ++j)
          for (int i = j; i < bk; ++i) C[j * BA_TB + i] -= C[k * BA_TB + i] * C[k * BA_TB + j];
      }
      double* Li = &Linv[(size_t)t.k * BA_TILE];  // column-major: Linv(r, c) at c*64 + r
      for (int c = 0; c < bk; ++c)
        for (int r = c; r < bk; ++r) {
          double s = (r == c) ? 1.0 : 0.0;
          for (int p = c; p < r; ++p) s -= C[p * BA_TB + r] * Li[c * BA_TB + p];
          Li[c * BA_TB + r] = s / C[r * BA_TB + r];
        }
      for (int r = 0; r < bk; ++r) {
        double s = 0;
        for (int p = 0; p <= r; ++p) s += Li[p * BA_TB + r] * b[(size_t)t.k * BA_TB + p];
        y[(size_t)t.k * BA_TB + r] = s;
      }
    } else if (t.type == BA_T_TRSM) {
      double* C = tile(S, t.tC);
      const double* Li = &Linv[(size_t)t.k * BA_TILE];
      const int bi = P.blkRows[t.i];
      std::vector<double> X((size_t)BA_TILE, 0.0);
      for (int r = 0; r < bi; ++r)
        for (int c = 0; c < bk; ++c) {
          double s = 0;
          for (int p = 0; p <= c; ++p) s += C[p * BA_TB + r] * Li[p * BA_TB + c];
          X[c * BA_TB + r] = s;
        }
      std::memcpy(C, X.data(), sizeof(double) * BA_TILE);
    } else if (t.type == BA_T_UPD) {
      double* C = tile(S, t.tC);
      const double* Ai = tile(S, t.tA);
      const double* Aj = tile(S, t.tB);
      const bool over = (t.flags & 2) != 0;
      if (over != (t.tC >= P.nTiles && cnt[t.tC] == 0)) {
        std::printf("FAIL: overwrite flag inconsistent\n");
        return 1;
      }
      for (int r = 0; r < BA_TB; ++r)
        for (int c = 0; c < BA_TB; ++c) {
          double s = 0;
          for (int p = 0; p < bk; ++p) s += Ai[p * BA_TB + r] * Aj[p * BA_TB + c];
          C[c * BA_TB + r] = (over ? 0.0 : C[c * BA_TB + r]) - s;
        }
      if (t.flags & 1) {
        double* bb = (t.l0 >= 0) ? &bS[(size_t)t.l0 * BA_TB] : &b[(size_t)t.i * BA_TB];
        if ((t.l0 >= 0) != (t.tC >= P.nTiles)) {
          std::printf("FAIL: rhs slot inconsistent\n");
          return 1;
        }
        for (int r = 0; r < BA_TB; ++r) {
          double s = 0;
          for (int p = 0; p < bk; ++p) s += Ai[p * BA_TB + r] * y[(size_t)t.k * BA_TB + p];
          bb[r] = (over ? 0.0 : bb[r]) - s;
        }
      }
    } else if (t.type == BA_T_SUM) {
      double* C = tile(S, t.tC);
      for (int e = t.l0; e < t.l1; ++e) {
        const BaSumEntry se = P.sumList[e];
        if (cnt[se.tile] < se.count) {
          std::printf("FAIL: SUM before its scratch tile %d is complete\n", se.tile);
          return 1;
        }
        const double* Sc = tile(S, se.tile);
        for (int q = 0; q < BA_TILE; ++q) C[q] += Sc[q];
        if (t.flags & 1)
          for (int r = 0; r < BA_TB; ++r) b[(size_t)t.i * BA_TB + r] += bS[(size_t)(se.tile - P.nTiles) * BA_TB + r];
      }
    } else {  // BWD
      std::vector<double> v(BA_TB);
      for (int p = 0; p < BA_TB; ++p) v[p] = y[(size_t)t.k * BA_TB + p];
      for (int e = t.l0; e < t.l1; ++e) {
        const BaBwdEntry be = P.bwdList[e];
        if (cnt[ntAll + be.blk] < 1) {
          std::printf("FAIL: BWD(%d) before x_%d\n", t.k, be.blk);
          return 1;
        }
        const double* L = tile(S, be.tile);
        for (int c = 0; c < bk; ++c) {
          double s = 0;
          for (int r = 0; r < P.blkRows[be.blk]; ++r) s += L[c * BA_TB + r] * x[(size_t)be.blk * BA_TB + r];
          v[c] -= s;
        }
      }
      const double* Li = &Linv[(size_t)t.k * BA_TILE];
      for (int p = 0; p < bk; ++p) {
        double s = 0;
        for (int c = p; c < bk; ++c) s += Li[p * BA_TB + c] * v[c];
        x[(size_t)t.k * BA_TB + p] = s;
      }
    }
    cnt[t.done] += 1;
  }
  // dense reference
  std::vector<double> Lr(A), xr(rhs);
  for (int k = 0; k < ns; ++k) {
    const double d = std::sqrt(Lr[(size_t)k * ns + k]);
    Lr[(size_t)k * ns + k] = d;
    for (int i = k + 1; i < ns; ++i) Lr[(size_t)i * ns + k] /= d;
    for (int j = k + 1; j < ns; ++j) {
      const double l = Lr[(size_t)j * ns + k];
      if (l == 0) continue;
      for (int i = j; i < ns; ++i) Lr[(size_t)i * ns + j] -= Lr[(size_t)i * ns + k] * l;
    }
  }
  for (int i = 0; i < ns; ++i) {
    double s = xr[i];
    for (int p = 0; p < i; ++p) s -= Lr[(size_t)i * ns + p] * xr[p];
    xr[i] = s / Lr[(size_t)i * ns + i];
  }
  for (int i = ns - 1; i >= 0; --i) {
    double s = xr[i];
    for (int p = i + 1; p < ns; ++p) s -= Lr[(size_t)p * ns + i] * xr[p];
    xr[i] = s / Lr[(size_t)i * ns + i];
  }
  double err = 0, nrm = 0;
  for (int a = 0; a < mf; ++a)
    for (int r = 0; r < 6; ++r) {
      const double xv = x[(size_t)P.camBlk[a] * BA_TB + P.camOff[a] + r];
      err = std::fmax(err, std::fabs(xv - xr[6 * a + r]));
      nrm = std::fmax(nrm, std::fabs(xr[6 * a + r]));
    }
  // SUM tasks of diagonal tiles (they also add the rhs parts of their scratch tiles) and BWD tasks
  // whose wait list is not a whole number of the kernel's chunks of 4
  int diagSums = 0, bwdNot4 = 0;
  for (const BaTask& t : P.tasks) {
    diagSums += (t.type == BA_T_SUM && (t.flags & 1)) ? 1 : 0;
    bwdNot4 += (t.type == BA_T_BWD && (t.l1 - t.l0) % 4 != 0) ? 1 : 0;
  }
  std::printf("{\"mf\": %d, \"nb\": %d, \"nd_depth\": %d, \"tiles_orig\": %d, \"tiles\": %d, \"scratch\": %d, "
              "\"tasks\": %d, \"critical_tasks\": %d, \"critical_cost\": %.1f, \"gflop\": %.4f, \"rel_err\": %.3e, "
              "\"diag_sums\": %d, \"bwd_not4\": %d}\n",
              mf, nb, P.ndDepth, P.nTilesOrig, P.nTiles, P.nScratch, (int)P.tasks.size(), P.criticalPathTasks,
              P.criticalPathCost, P.flops * 1e-9, err / nrm, diagSums, bwdNot4);
  if (!(err / nrm < 1e-9)) {
    std::printf("FAIL: solution differs\n");
    return 1;
  }
  std::printf("OK\n");
  return 0;
}
