/* posegraph_general_oracle.cpp -- CPU restatement of the camera-group merge's pose-graph solve (TEST
 * INFRASTRUCTURE ONLY; nothing under coslam_b200/ may call it).  Built by oracle/Makefile.pg_general into
 * oracle/liboracle_pg_general.so.
 *
 * PINNED: tests/test_posegraph_general.py compares it with the UNMODIFIED reference
 * (oracle/_ref/libposegraph_merge_ref.so, live where it is built) and with
 * tests/golden/posegraph_merge_ref.npz generated from it.
 *
 * The post-BA restatement (posegraph_oracle.cpp) is compiled into this translation unit unchanged, so
 * both share its Frobenius-nearest rotation (polar iteration), the projection step of :205-211. */
#include <algorithm>

#include "posegraph_oracle.cpp"

/* ===================================================================================================
 * General edge sets with shared unknown scales: GlobalPoseGraph::computeNewCameraRotations (:52-218)
 * + ::computeNewCameraTranslations4 (:361-525), scale columns given per edge (-1 = known scale).
 * The dense solve above does not scale to thousands of nodes; here the normal equations of each system
 * are factored in ENVELOPE (skyline) storage in the natural column order -- per free node its three
 * components, the scale columns last -- which keeps chains, key-frame grids and loop closures cheap,
 * again followed by one refinement step.  The three rotation systems (one per column of R_k, :96-134)
 * share one matrix and are solved as three right-hand sides.
 * =================================================================================================== */
namespace {

struct SpRow {
  int n = 0;
  int col[5];
  double val[5];
  void add(int c, double v) { col[n] = c; val[n++] = v; }
};

/* X (n x nrhs, row-major) = argmin |A X - B| for the sparse rows A; false on a non-positive pivot */
bool lstsq_envelope(int n, const std::vector<SpRow>& A, const std::vector<double>& B, int nrhs,
                    std::vector<double>& X) {
  const int m = (int)A.size();
  X.assign((size_t)n * nrhs, 0.0);
  if (n == 0) return true;
  std::vector<int> first(n);
  for (int c = 0; c < n; ++c) first[c] = c;
  for (const SpRow& r : A) {
    int lo = n;
    for (int q = 0; q < r.n; ++q) lo = std::min(lo, r.col[q]);
    for (int q = 0; q < r.n; ++q) first[r.col[q]] = std::min(first[r.col[q]], lo);
  }
  std::vector<size_t> off(n + 1, 0); /* row i holds columns first[i] .. i */
  for (int i = 0; i < n; ++i) off[i + 1] = off[i] + (size_t)(i - first[i] + 1);
  std::vector<double> G(off[n], 0.0);
  auto at = [&](int i, int j) -> double& { return G[off[i] + (size_t)(j - first[i])]; };
  for (const SpRow& r : A)
    for (int a = 0; a < r.n; ++a)
      for (int b = 0; b < r.n; ++b)
        if (r.col[a] >= r.col[b]) at(r.col[a], r.col[b]) += r.val[a] * r.val[b];
  for (int i = 0; i < n; ++i) { /* row-oriented envelope Cholesky, in place */
    for (int j = first[i]; j <= i; ++j) {
      double s = at(i, j);
      for (int k = std::max(first[i], first[j]); k < j; ++k) s -= at(i, k) * at(j, k);
      if (j < i) {
        at(i, j) = s / at(j, j);
      } else {
        if (!(s > 0)) return false;
        at(i, i) = std::sqrt(s);
      }
    }
  }
  std::vector<double> res(B), g(n), y(n);
  for (int pass = 0; pass < 2; ++pass) {
    for (int h = 0; h < nrhs; ++h) {
      std::fill(g.begin(), g.end(), 0.0);
      for (int r = 0; r < m; ++r)
        for (int q = 0; q < A[r].n; ++q) g[A[r].col[q]] += A[r].val[q] * res[(size_t)r * nrhs + h];
      for (int i = 0; i < n; ++i) {
        double s = g[i];
        for (int k = first[i]; k < i; ++k) s -= at(i, k) * y[k];
        y[i] = s / at(i, i);
      }
      for (int i = n - 1; i >= 0; --i) {
        y[i] /= at(i, i);
        for (int k = first[i]; k < i; ++k) y[k] -= at(i, k) * y[i];
      }
      for (int i = 0; i < n; ++i) X[(size_t)i * nrhs + h] += y[i];
    }
    for (int r = 0; r < m; ++r)
      for (int h = 0; h < nrhs; ++h) {
        double s = B[(size_t)r * nrhs + h];
        for (int q = 0; q < A[r].n; ++q) s -= A[r].val[q] * X[(size_t)A[r].col[q] * nrhs + h];
        res[(size_t)r * nrhs + h] = s;
      }
  }
  return true;
}

}  // namespace

/* Returns 0, 1 when a normal matrix has a non-positive pivot (rank deficient), 2 on bad indices. */
extern "C" int orc_posegraph_solve(int nNodes, const int* fixed, const double* R, const double* t, int nEdges,
                                   const int* id1, const int* id2, const double* eR, const double* et,
                                   const int* scaleCol, int nScale, double* newR, double* newt, double* scale) {
  std::vector<int> colOf(nNodes, -1);
  int nF = 0;
  for (int k = 0; k < nNodes; ++k)
    if (!fixed[k]) colOf[k] = nF++;
  for (int e = 0; e < nEdges; ++e) {
    const int c = scaleCol ? scaleCol[e] : -1;
    if (id1[e] < 0 || id1[e] >= nNodes || id2[e] < 0 || id2[e] >= nNodes || id1[e] == id2[e] || c < -1 ||
        c >= nScale)
      return 2;
  }
  std::vector<SpRow> A;
  std::vector<double> bR, bT;
  for (int e = 0; e < nEdges; ++e) {
    const int i = id1[e], j = id2[e], c = scaleCol ? scaleCol[e] : -1;
    if (fixed[i] && fixed[j]) continue; /* (:59, :368) */
    const double* Rij = eR + 9 * (size_t)e;
    const double* tij = et + 3 * (size_t)e;
    for (int u = 0; u < 3; ++u) {
      SpRow row;
      if (!fixed[j]) row.add(3 * colOf[j] + u, 1.0);
      if (!fixed[i])
        for (int v = 0; v < 3; ++v) row.add(3 * colOf[i] + v, -Rij[3 * u + v]);
      /* rotations, column a: col_a(R_j) - R_ij col_a(R_i) = 0 (:82-195) */
      for (int a = 0; a < 3; ++a) {
        double rhs = 0.0;
        if (fixed[j]) rhs -= R[9 * (size_t)j + 3 * u + a];
        if (fixed[i])
          for (int v = 0; v < 3; ++v) rhs += Rij[3 * u + v] * R[9 * (size_t)i + 3 * v + a];
        bR.push_back(rhs);
      }
      /* translations: t_j - R_ij t_i - s_c t_ij = 0, or = t_ij for a known scale (:417-500) */
      double rhs = c < 0 ? tij[u] : 0.0;
      if (fixed[j]) rhs -= t[3 * (size_t)j + u];
      if (fixed[i])
        for (int v = 0; v < 3; ++v) rhs += Rij[3 * u + v] * t[3 * (size_t)i + v];
      bT.push_back(rhs);
      A.push_back(row);
    }
  }
  std::vector<double> xR, xT;
  if (!lstsq_envelope(3 * nF, A, bR, 3, xR)) return 1;
  {
    /* the translation rows carry the scale column as a fifth entry */
    int r = 0;
    for (int e = 0; e < nEdges; ++e) {
      const int i = id1[e], j = id2[e], c = scaleCol ? scaleCol[e] : -1;
      if (fixed[i] && fixed[j]) continue;
      for (int u = 0; u < 3; ++u, ++r)
        if (c >= 0) A[r].add(3 * nF + c, -et[3 * (size_t)e + u]);
    }
  }
  if (!lstsq_envelope(3 * nF + nScale, A, bT, 1, xT)) return 1;
  for (int k = 0; k < nNodes; ++k) {
    if (colOf[k] < 0) {
      std::memcpy(newR + 9 * (size_t)k, R + 9 * (size_t)k, 72);
      std::memcpy(newt + 3 * (size_t)k, t + 3 * (size_t)k, 24);
      continue;
    }
    double M[9];
    for (int u = 0; u < 3; ++u)
      for (int a = 0; a < 3; ++a) M[3 * u + a] = xR[(size_t)(3 * colOf[k] + u) * 3 + a];
    nearest_rotation(M, newR + 9 * (size_t)k);
    std::memcpy(newt + 3 * (size_t)k, &xT[3 * (size_t)colOf[k]], 24);
  }
  for (int c = 0; c < nScale; ++c) scale[c] = xT[3 * (size_t)nF + c];
  return 0;
}
