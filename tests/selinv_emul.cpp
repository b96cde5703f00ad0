// selinv_emul.cpp -- CPU check of the selected-inversion plan of coslam_b200/csrc/ba_plan.h (test
// infrastructure).  Builds the same random SPD reduced camera systems as plan_emul.cpp, factors the permuted
// system densely, places the factor into the plan's tiles (asserting that it has no entry outside them: the
// tile pattern is closed under fill), then executes ba_make_selinv_plan's steps SEQUENTIALLY -- asserting that
// every operand tile of a task is final when its turn comes -- and writes S and the resulting Z (camera
// order, pattern blocks only) for tests/test_ba_selinv_plan.py to compare with numpy.linalg.inv(S).
//   usage: selinv_emul <outdir> <mf> <pattern: band|dense|random> <param> [ndDepth]
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>

#include "../coslam_b200/csrc/ba_plan.h"

using namespace coslam;

static int fail(const char* msg) {
  std::printf("FAIL: %s\n", msg);
  return 1;
}

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  const std::string dir = argv[1];
  const int mf = std::atoi(argv[2]);
  const std::string pat = argv[3];
  const double param = std::atof(argv[4]);
  const int depth = argc > 5 ? std::atoi(argv[5]) : -1;
  std::mt19937_64 rng(1234 + mf);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::vector<uint8_t> adj((size_t)mf * mf, 0);
  for (int a = 0; a < mf; ++a)
    for (int b = a; b < mf; ++b) {
      bool on = (a == b);
      if (pat == "band") on = on || (b - a) <= (int)param;
      if (pat == "dense") on = true;
      if (pat == "random") on = on || (std::abs(U(rng)) < param) || (b - a) <= 2;
      if (pat == "split") on = on || ((b - a) <= (int)param && (a < mf / 2) == (b < mf / 2));  // two components
      adj[(size_t)a * mf + b] = adj[(size_t)b * mf + a] = on ? 1 : 0;
    }
  const int ns = 6 * mf;
  std::vector<double> A((size_t)ns * ns, 0.0);
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
  }
  const BaPlan P = ba_make_plan(mf, adj, depth);
  const BaSelPlan SP = ba_make_selinv_plan(P);
  const int nb = P.nb;
  // permuted order: row of camera a, parameter r = 64 * block + offset (padding rows unused)
  std::vector<int> pos(ns);
  for (int a = 0; a < mf; ++a)
    for (int r = 0; r < 6; ++r) pos[6 * a + r] = BA_TB * P.camBlk[a] + P.camOff[a] + r;
  const int np = BA_TB * nb;
  std::vector<double> L((size_t)np * np, 0.0);
  std::vector<uint8_t> used(np, 0);
  for (int i = 0; i < ns; ++i) {
    used[pos[i]] = 1;
    for (int j = 0; j < ns; ++j) L[(size_t)pos[i] * np + pos[j]] = A[(size_t)i * ns + j];
  }
  for (int k = 0; k < np; ++k) {
    if (!used[k]) continue;
    const double d = std::sqrt(L[(size_t)k * np + k]);
    L[(size_t)k * np + k] = d;
    for (int i = k + 1; i < np; ++i) L[(size_t)i * np + k] /= d;
    for (int j = k + 1; j < np; ++j) {
      const double l = L[(size_t)j * np + k];
      if (l == 0) continue;
      for (int i = j; i < np; ++i) L[(size_t)i * np + j] -= L[(size_t)i * np + k] * l;
    }
  }
  // the factor's tiles (column-major, as on the device); nothing of L may fall outside them
  auto T = [&](int i, int j) { return P.tileIdx[(size_t)i * nb + j]; };
  std::vector<double> Lt((size_t)P.nTiles * BA_TILE, 0.0), Z((size_t)P.nTiles * BA_TILE, 0.0);
  for (int i = 0; i < np; ++i)
    for (int j = 0; j <= i; ++j) {
      const double v = L[(size_t)i * np + j];
      if (v == 0.0) continue;
      const int t = T(i / BA_TB, j / BA_TB);
      if (t < 0) return fail("factor entry outside the tile pattern");
      Lt[(size_t)t * BA_TILE + (j % BA_TB) * BA_TB + i % BA_TB] = v;
    }
  auto el = [](std::vector<double>& v, int t, int r, int c) -> double& {
    return v[(size_t)t * BA_TILE + (size_t)c * BA_TB + r];
  };
  // X_k = L_kk^-T (upper triangular), dense per block
  std::vector<std::vector<double>> X(nb);
  for (int k = 0; k < nb; ++k) {
    const int bk = P.blkRows[k], t = T(k, k);
    std::vector<double> Li((size_t)bk * bk, 0.0);  // L_kk^-1, row-major
    for (int c = 0; c < bk; ++c)
      for (int r = c; r < bk; ++r) {
        double s = (r == c) ? 1.0 : 0.0;
        for (int p = c; p < r; ++p) s -= el(Lt, t, r, p) * Li[(size_t)p * bk + c];
        Li[(size_t)r * bk + c] = s / el(Lt, t, r, r);
      }
    X[k].assign((size_t)bk * bk, 0.0);
    for (int r = 0; r < bk; ++r)
      for (int c = 0; c < bk; ++c) X[k][(size_t)r * bk + c] = Li[(size_t)c * bk + r];
  }
  // the plan, one step after the other, every task on final operands only
  std::vector<uint8_t> fin(P.nTiles, 0);
  if ((int)SP.stepBegin.size() != nb + 1) return fail("one step per pivot");
  for (int q = 0; q < nb; ++q) {
    const int t0 = SP.stepBegin[q], t1 = SP.stepBegin[q + 1];
    if (t1 <= t0) return fail("empty step");
    for (int ti = t0; ti < t1; ++ti) {
      const BaSelTask& t = SP.tasks[ti];
      if (t.k != nb - 1 - q || (t.i == t.k) != (ti == t1 - 1)) return fail("task out of place");
      const int k = t.k, bk = P.blkRows[k], bi = P.blkRows[t.i];
      std::vector<double> G((size_t)BA_TB * BA_TB, 0.0);  // row-major bi x bk (off-diagonal) or bk x bk
      for (int o = t.opBegin; o < t.opEnd; ++o) {
        const BaSelOp& op = SP.ops[o];
        if (op.tZ < 0 || op.tL < 0 || !fin[op.tZ]) return fail("operand tile not final");
        if (op.tL != T(op.j, k)) return fail("wrong factor operand");
        const int bj = P.blkRows[op.j];
        if (t.i != k) {  // G += Z_ij L_jk
          for (int r = 0; r < bi; ++r)
            for (int c = 0; c < bk; ++c) {
              double s = 0;
              for (int p = 0; p < bj; ++p)
                s += (op.zT ? el(Z, op.tZ, p, r) : el(Z, op.tZ, r, p)) * el(Lt, op.tL, p, c);
              G[(size_t)r * bk + c] += s;
            }
        } else {  // G += L_jk^T Z_jk
          for (int r = 0; r < bk; ++r)
            for (int c = 0; c < bk; ++c) {
              double s = 0;
              for (int p = 0; p < bj; ++p) s += el(Lt, op.tL, p, r) * el(Z, op.tZ, p, c);
              G[(size_t)r * bk + c] += s;
            }
        }
      }
      const std::vector<double>& Xk = X[k];
      if (t.i != k) {  // Z_ik = -G L_kk^-1 = -G X_k^T
        for (int r = 0; r < bi; ++r)
          for (int c = 0; c < bk; ++c) {
            double s = 0;
            for (int p = 0; p < bk; ++p) s += G[(size_t)r * bk + p] * Xk[(size_t)c * bk + p];
            el(Z, t.tOut, r, c) = -s;
          }
      } else {  // Z_kk = X_k (X_k^T - G)
        for (int r = 0; r < bk; ++r)
          for (int c = 0; c < bk; ++c) {
            double s = 0;
            for (int p = 0; p < bk; ++p) s += Xk[(size_t)r * bk + p] * (Xk[(size_t)c * bk + p] - G[(size_t)p * bk + c]);
            el(Z, t.tOut, r, c) = s;
          }
      }
      fin[t.tOut] = 1;
    }
  }
  for (int t = 0; t < P.nTiles; ++t)
    if (!fin[t]) return fail("a tile of the pattern was never computed");
  // S and Z in camera order; Z on the pattern blocks (both triangles), mask[a][c] = 1 there
  std::vector<double> Zd((size_t)ns * ns, 0.0);
  std::vector<uint8_t> mask((size_t)mf * mf, 0);
  for (int a = 0; a < mf; ++a)
    for (int c = 0; c < mf; ++c) {
      const int ba = P.camBlk[a], bc = P.camBlk[c];
      const int t = ba >= bc ? T(ba, bc) : T(bc, ba);
      if (t < 0) continue;
      mask[(size_t)a * mf + c] = 1;
      for (int r = 0; r < 6; ++r)
        for (int q = 0; q < 6; ++q) {
          const int pr = pos[6 * a + r] % BA_TB, pq = pos[6 * c + q] % BA_TB;
          const bool lower = ba > bc || (ba == bc && pr >= pq);
          Zd[(size_t)(6 * a + r) * ns + 6 * c + q] = lower ? el(Z, t, pr, pq) : el(Z, t, pq, pr);
        }
    }
  auto dump = [&](const char* name, const void* p, size_t bytes) {
    FILE* f = std::fopen((dir + "/" + name).c_str(), "wb");
    if (!f) return false;
    const bool ok = std::fwrite(p, 1, bytes, f) == bytes;
    std::fclose(f);
    return ok;
  };
  if (!dump("S.bin", A.data(), 8 * A.size()) || !dump("Z.bin", Zd.data(), 8 * Zd.size()) ||
      !dump("mask.bin", mask.data(), mask.size()))
    return fail("cannot write the output files");
  std::printf("{\"mf\": %d, \"nb\": %d, \"nd_depth\": %d, \"tiles\": %d, \"steps\": %d, \"tasks\": %d, \"ops\": %d}\n",
              mf, nb, P.ndDepth, P.nTiles, (int)SP.stepBegin.size() - 1, (int)SP.tasks.size(), (int)SP.ops.size());
  std::printf("OK\n");
  return 0;
}
