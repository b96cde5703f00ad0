// ba_plan.h -- host-side planning of the reduced-camera-system solve (plain C++, no CUDA).
//
// The reduced camera system S of a bundle adjustment (BA-4 step iv/v, SURVEY.md 8a; the reference
// hands it to LAPACK inside sba_motstr_levmar_x, call app/SL_CoSLAMBA.cpp:360-363) is symmetric
// positive definite with one 6x6 block per pair of co-visible free cameras.  This header turns the
// camera co-visibility into everything the device solver (ba_tile.cuh) needs:
//
//   1. an ORDERING of the free cameras.  Sequential key frames give a banded S; a banded Cholesky is
//      one long chain of dependent pivots.  Nested dissection cuts the chain: separators as wide as
//      the band decouple the interiors, which are then eliminated concurrently (each from both of
//      its ends), and only the small separator systems remain sequential.  Non-band-like
//      co-visibility (local BA, inter-camera pose) keeps the natural order.
//   2. a BLOCKING of the ordered cameras into blocks of <= 10 cameras (<= 60 rows) that never
//      straddle a region, stored as 64x64 column-major TILES (block-sparse, lower triangle, only
//      structurally non-zero tiles incl. Cholesky fill).
//   3. the TASK DAG of a right-looking tile Cholesky + both substitutions:
//        POTRF(k)   : factor tile (k,k), invert the factor, y_k = Linv_k b_k
//        TRSM(i,k)  : L_ik = A_ik Linv_k^T
//        UPD(i,j,k) : A_ij -= L_ik L_jk^T   (i == j: also b_i -= L_ik y_k)
//        BWD(k)     : x_k = Linv_k^T (y_k - sum_i L_ik^T x_i)
//        SUM(i,j)   : A_ij += sum_g scratch_g(i,j)   (multifrontal-style extend-add, see below)
//      with per-tile completion counters (the updates of one tile are applied in ONE fixed order,
//      so the result is deterministic) and a critical-path-first (bottom-level) list order that
//      is also a topological order: CTAs take tasks by an atomic ticket and spin on the counters,
//      which cannot deadlock because every dependency of a task precedes it in the list.
//      A separator tile receives an update from every block of every region below it; applied to
//      the tile itself they would form one chain of ~nb read-modify-writes.  Updates whose pivot
//      block lies in ANOTHER region than the target column are therefore accumulated in a scratch
//      tile private to (target tile, pivot region) -- the regions proceed concurrently -- and one
//      SUM task adds the scratch tiles to the target in a fixed order.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace coslam {

constexpr int BA_TB = 64;                  // tile edge (storage)
constexpr int BA_TILE = BA_TB * BA_TB;     // doubles per tile
constexpr int BA_BLK_CAMS = 10;            // cameras per block (60 of the 64 tile rows are used)

enum BaTaskType { BA_T_POTRF = 0, BA_T_TRSM = 1, BA_T_UPD = 2, BA_T_BWD = 3, BA_T_SUM = 4 };

struct BaTask {  // 64 bytes, read by every thread of the CTA that executes it
  // flags bit 0: diagonal tile (UPD with i == j / SUM of a diagonal tile) -> also handles b_i;
  //       bit 1: UPD is the first one into a scratch tile -> overwrite instead of accumulate
  int type, k, i, flags;
  int tC, tA, tB;         // tile indices: output tile; UPD: (i,k), (j,k); TRSM: tA = Linv index k
  int done;               // counter incremented on completion
  int w0i, w0v, w1i, w1v, w2i, w2v;  // wait until cnt[w?i] >= w?v (w?i < 0: unused)
  // BWD: range in BaPlan::bwdList; SUM: range in BaPlan::sumList;
  // UPD: l0 = scratch slot whose rhs vector receives the b_i part (-1: the real rhs of block i)
  int l0, l1;
};

struct BaBwdEntry {
  int blk;   // block row i of struct(k)
  int tile;  // tile index of (i, k)
  int fin;   // value of the tile's counter when L_ik is final (all updates + its TRSM)
  int pad;
};

struct BaSumEntry {
  int tile;   // scratch tile (index into the tile array, >= nTiles)
  int count;  // updates it receives (its counter must reach this value)
};

struct BaPlan {
  int mf = 0, nb = 0;
  int ndDepth = 0;
  std::vector<int> order;    // order[pos] = free camera at position pos of the elimination order
  std::vector<int> camBlk;   // per free camera: block
  std::vector<int> camOff;   // per free camera: row offset inside the block (multiple of 6)
  std::vector<int> blkRows;  // rows used in block k (multiple of 6, <= 60)
  std::vector<int> blkCam0;  // first position (in `order`) of block k; blkCam0[nb] = mf
  std::vector<int> tileIdx;  // nb*nb: tileIdx[i*nb + j], i >= j; -1 = structurally zero
  int nTilesOrig = 0;        // tiles the Schur contraction can touch (incl. all diagonal tiles)
  int nTiles = 0;            // + fill
  int nScratch = 0;          // scratch tiles (tile indices nTiles .. nTiles + nScratch - 1)
  std::vector<int> blkRegion;
  std::vector<BaSumEntry> sumList;
  std::vector<BaTask> tasks; // in execution (ticket) order
  std::vector<BaBwdEntry> bwdList;
  int nCounters = 0;         // (nTiles + nScratch) tile counters + nb "x_k done" counters
  double flops = 0;          // 2 * (multiply-adds of the tile tasks, counted on the used rows)
  int criticalPathTasks = 0; // length (in tasks) of the longest dependency chain
  double criticalPathCost = 0;
};

namespace plan_detail {

// splits `n` consecutive positions into ceil(n / BA_BLK_CAMS) blocks of nearly equal size
inline void split_blocks(int first, int n, std::vector<std::pair<int, int>>& out) {
  if (n <= 0) return;
  const int q = (n + BA_BLK_CAMS - 1) / BA_BLK_CAMS;
  int at = first;
  for (int b = 0; b < q; ++b) {
    const int len = n / q + (b < n % q ? 1 : 0);
    out.push_back({at, len});
    at += len;
  }
}

struct Region {
  int lo, hi;
  bool separator;
};

// hiN[a] = largest neighbour index of camera a in the natural order (>= a)
inline void nd_recurse(int lo, int hi, int depth, const std::vector<int>& hiN, int bw,
                       std::vector<Region>& out) {
  const int len = hi - lo;
  if (depth <= 0 || len < 3 * bw + 2 * BA_BLK_CAMS) {
    out.push_back({lo, hi, false});
    return;
  }
  int s0 = lo + (len - bw) / 2;
  if (s0 <= lo) {
    out.push_back({lo, hi, false});
    return;
  }
  // the separator must swallow every camera that sees something left of it
  int s1 = s0;
  for (int a = lo; a < s0; ++a) s1 = std::max(s1, hiN[a] + 1);
  s1 = std::max(s1, s0 + 1);
  if (s1 >= hi) {
    out.push_back({lo, hi, false});
    return;
  }
  nd_recurse(lo, s0, depth - 1, hiN, bw, out);
  nd_recurse(s1, hi, depth - 1, hiN, bw, out);
  out.push_back({s0, s1, true});
}

}  // namespace plan_detail

// adj: mf*mf, adj[a*mf + b] != 0 iff free cameras a and b share a point (symmetric; the diagonal
// is implied).  ndDepthOverride < 0: choose the dissection depth automatically.
inline BaPlan ba_make_plan(int mf, const std::vector<uint8_t>& adj, int ndDepthOverride = -1) {
  using namespace plan_detail;
  BaPlan P;
  P.mf = mf;
  if (mf <= 0) return P;
  // ---- 1. ordering -----------------------------------------------------------------------
  std::vector<int> hiN(mf);
  int bw = 0;
  for (int a = 0; a < mf; ++a) {
    int h = a;
    for (int b = mf - 1; b > a; --b)
      if (adj[(size_t)a * mf + b] || adj[(size_t)b * mf + a]) {
        h = b;
        break;
      }
    hiN[a] = h;
    bw = std::max(bw, h - a);
  }
  const int sepw = bw + 1;
  const bool bandLike = (mf >= 4 * sepw && mf > 6 * BA_BLK_CAMS);
  int depth = 0;
  if (ndDepthOverride >= 0) {
    depth = bandLike ? ndDepthOverride : 0;
  } else if (bandLike) {
    // estimate of the critical path in block steps: half a leaf interior (two-sided elimination)
    // + one separator per level
    const double sepBlocks = (double)((sepw + BA_BLK_CAMS - 1) / BA_BLK_CAMS);
    double best = 1e30;
    for (int d = 0; d <= 5; ++d) {
      const double leaves = (double)(1 << d);
      const double interior = (mf - (leaves - 1) * sepw) / leaves;
      if (interior < 2.0 * BA_BLK_CAMS) break;
      const double path = interior / BA_BLK_CAMS / 2.0 + d * sepBlocks;
      if (path < best - 0.75) {  // deeper only if it buys most of a block step (more fill otherwise)
        best = path;
        depth = d;
      }
    }
  }
  P.ndDepth = depth;
  std::vector<Region> regions;
  nd_recurse(0, mf, depth, hiN, sepw, regions);
  // blocks: interiors are eliminated from both ends towards the middle, separators front to back
  std::vector<std::pair<int, int>> blocks;  // (first natural index, count) in elimination order
  std::vector<int> blockRegion;
  for (size_t ri = 0; ri < regions.size(); ++ri) {
    const Region& r = regions[ri];
    std::vector<std::pair<int, int>> nat;
    split_blocks(r.lo, r.hi - r.lo, nat);
    for (size_t q = 0; q < nat.size(); ++q) blockRegion.push_back((int)ri);
    if (r.separator || !bandLike) {
      for (auto& b : nat) blocks.push_back(b);
    } else {
      // two-sided: B0, Bq-1, B1, Bq-2, ... (the fill stays inside the band only for band-like S)
      int a = 0, z = (int)nat.size() - 1;
      while (a <= z) {
        blocks.push_back(nat[a]);
        if (z != a) blocks.push_back(nat[z]);
        ++a;
        --z;
      }
    }
  }
  const int nb = (int)blocks.size();
  P.nb = nb;
  P.order.resize(mf);
  P.camBlk.assign(mf, 0);
  P.camOff.assign(mf, 0);
  P.blkRows.assign(nb, 0);
  P.blkCam0.assign(nb + 1, 0);
  P.blkRegion = blockRegion;
  {
    int pos = 0;
    for (int k = 0; k < nb; ++k) {
      P.blkCam0[k] = pos;
      for (int c = 0; c < blocks[k].second; ++c) {
        const int cam = blocks[k].first + c;
        P.order[pos++] = cam;
        P.camBlk[cam] = k;
        P.camOff[cam] = 6 * c;
      }
      P.blkRows[k] = 6 * blocks[k].second;
    }
    P.blkCam0[nb] = pos;
  }
  // ---- 2. block structure + symbolic fill -------------------------------------------------
  std::vector<uint8_t> st((size_t)nb * nb, 0);  // st[i*nb + j], i >= j
  for (int k = 0; k < nb; ++k) st[(size_t)k * nb + k] = 1;
  for (int a = 0; a < mf; ++a)
    for (int b = a + 1; b < mf; ++b)
      if (adj[(size_t)a * mf + b] || adj[(size_t)b * mf + a]) {
        const int i = std::max(P.camBlk[a], P.camBlk[b]), j = std::min(P.camBlk[a], P.camBlk[b]);
        st[(size_t)i * nb + j] = 1;
      }
  P.tileIdx.assign((size_t)nb * nb, -1);
  int nt = 0;
  for (int j = 0; j < nb; ++j)
    for (int i = j; i < nb; ++i)
      if (st[(size_t)i * nb + j]) P.tileIdx[(size_t)i * nb + j] = nt++;
  P.nTilesOrig = nt;
  std::vector<std::vector<int>> strct(nb);
  for (int k = 0; k < nb; ++k) {
    for (int i = k + 1; i < nb; ++i)
      if (st[(size_t)i * nb + k]) strct[k].push_back(i);
    const auto& s = strct[k];
    for (size_t a = 0; a < s.size(); ++a)
      for (size_t b = a + 1; b < s.size(); ++b) st[(size_t)s[b] * nb + s[a]] = 1;  // fill (i > j)
  }
  for (int j = 0; j < nb; ++j)
    for (int i = j; i < nb; ++i)
      if (st[(size_t)i * nb + j] && P.tileIdx[(size_t)i * nb + j] < 0) P.tileIdx[(size_t)i * nb + j] = nt++;
  P.nTiles = nt;
  // ---- 3. tasks ------------------------------------------------------------------------------
  // Generated pivot by pivot.  The updates of one tile commute mathematically but must be applied
  // in ONE fixed order (determinism, and no two CTAs may read-modify-write a tile at once).  Pivot
  // order would serialise a separator tile behind the slowest interior; instead the order follows
  // the estimated time at which each update's operands become available (pass 1 below).
  auto T = [&](int i, int j) { return P.tileIdx[(size_t)i * nb + j]; };
  const bool useScratch = regions.size() > 1;
  // scratch slot per (target tile, pivot region): created on first use
  std::vector<std::vector<std::pair<int, int>>> scratchOf(nt);  // target tile -> (region, scratch tile)
  int nScratch = 0;
  auto scratchTile = [&](int tile, int region) {
    for (auto& e : scratchOf[tile])
      if (e.first == region) return e.second;
    scratchOf[tile].push_back({region, nt + nScratch});
    return nt + nScratch++;
  };
  std::vector<BaTask> gen;
  std::vector<std::vector<int>> preds;  // predecessor task ids
  std::vector<double> cost;
  std::vector<std::vector<int>> tileUpd;  // UPD task ids per output tile (real and scratch)
  tileUpd.resize(nt);
  std::vector<int> finalTask(nt, -1);     // POTRF / TRSM task of a real tile
  std::vector<int> potrfTask(nb, -1), bwdTask(nb, -1);
  auto blank = [] {
    BaTask t;
    t.type = t.k = t.i = t.flags = 0;
    t.tC = t.tA = t.tB = t.done = -1;
    t.w0i = t.w1i = t.w2i = -1;
    t.w0v = t.w1v = t.w2v = 0;
    t.l0 = t.l1 = 0;
    return t;
  };
  const double cPotrf = 9.0, cTrsm = 4.0, cUpd = 4.0, cBwd = 3.0, cSum = 2.0;
  auto push = [&](const BaTask& t, double c) {
    gen.push_back(t);
    cost.push_back(c);
    preds.push_back({});
    return (int)gen.size() - 1;
  };
  for (int k = 0; k < nb; ++k) {
    const int tkk = T(k, k);
    {
      BaTask t = blank();
      t.type = BA_T_POTRF;
      t.k = t.i = k;
      t.tC = t.done = t.w0i = tkk;
      potrfTask[k] = finalTask[tkk] = push(t, cPotrf);
      const double r = P.blkRows[k];
      P.flops += 2.0 * (r * r * r / 3.0 + r * r * r / 3.0);
    }
    const auto& s = strct[k];
    std::vector<int> trsmTask(s.size());
    for (size_t a = 0; a < s.size(); ++a) {
      const int i = s[a], tik = T(i, k);
      BaTask t = blank();
      t.type = BA_T_TRSM;
      t.k = k;
      t.i = i;
      t.tC = t.done = t.w0i = tik;
      t.tA = k;
      t.w1i = tkk;
      trsmTask[a] = finalTask[tik] = push(t, cTrsm);
      preds[trsmTask[a]].push_back(potrfTask[k]);
      P.flops += 2.0 * P.blkRows[i] * (double)P.blkRows[k] * P.blkRows[k];
    }
    for (size_t b = 0; b < s.size(); ++b)
      for (size_t a = b; a < s.size(); ++a) {
        const int i = s[a], j = s[b], tij = T(i, j);
        int target = tij;
        if (useScratch && P.blkRegion[k] != P.blkRegion[j]) {
          target = scratchTile(tij, P.blkRegion[k]);
          if ((int)tileUpd.size() <= target) tileUpd.resize(target + 1);
        }
        BaTask t = blank();
        t.type = BA_T_UPD;
        t.k = k;
        t.i = i;
        t.flags = (i == j) ? 1 : 0;
        t.tC = t.done = t.w0i = target;
        t.tA = t.w1i = T(i, k);
        t.tB = t.w2i = T(j, k);
        t.l0 = (target == tij) ? -1 : target - nt;
        const int id = push(t, cUpd);
        preds[id].push_back(trsmTask[a]);
        if (a != b) preds[id].push_back(trsmTask[b]);
        tileUpd[target].push_back(id);
        P.flops += 2.0 * P.blkRows[i] * (double)P.blkRows[j] * P.blkRows[k];
      }
  }
  P.nScratch = nScratch;
  const int ntAll = nt + nScratch;
  tileUpd.resize(ntAll);
  P.nCounters = ntAll + nb;
  // SUM tasks: one per real tile that owns scratch tiles (generated after its contributors; the
  // topological sort below puts it in place)
  std::vector<int> sumTask(nt, -1);
  for (int tl = 0; tl < nt; ++tl) {
    if (scratchOf[tl].empty()) continue;
    BaTask t = blank();
    t.type = BA_T_SUM;
    t.tC = t.done = t.w0i = tl;
    t.w0v = 0;
    // block coordinates of the tile (for the rhs of diagonal tiles)
    sumTask[tl] = push(t, cSum);
  }
  for (int j = 0; j < nb; ++j)
    for (int i = j; i < nb; ++i) {
      const int tl = T(i, j);
      if (tl >= 0 && sumTask[tl] >= 0) {
        gen[sumTask[tl]].i = i;
        gen[sumTask[tl]].k = j;
        gen[sumTask[tl]].flags = (i == j) ? 1 : 0;
      }
    }
  const int nFactorTasks = (int)gen.size();
  // pass 1: earliest finish with unlimited workers, updates of a tile treated as independent.
  // Generation order is topological for POTRF/TRSM/UPD; SUM tasks sit at the end of `gen` but only
  // depend on UPDs and only feed tasks of later pivots, so they are evaluated on demand.
  std::vector<double> est(nFactorTasks, -1.0);
  auto updDone = [&](int tile) {  // time when every update (and the SUM) of a real tile is in
    double st = 0;
    for (int u : tileUpd[tile]) st = std::max(st, est[u]);
    if (sumTask[tile] >= 0) {
      double ss = 0;
      for (auto& e : scratchOf[tile])
        for (int u : tileUpd[e.second]) ss = std::max(ss, est[u]);
      est[sumTask[tile]] = ss + cSum;
      st = std::max(st, est[sumTask[tile]]);
    }
    return st;
  };
  for (int t = 0; t < nFactorTasks; ++t) {
    if (gen[t].type == BA_T_SUM) continue;
    double st = 0;
    for (int p : preds[t]) st = std::max(st, est[p]);
    if (gen[t].type != BA_T_UPD) st = std::max(st, updDone(gen[t].tC));
    est[t] = st + cost[t];
  }
  // sequence the updates of every tile by operand-ready time; final wait values.  A real tile
  // with scratch tiles takes its SUM as update number 0.
  std::vector<int> nupd(ntAll, 0);
  for (int tl = 0; tl < ntAll; ++tl) {
    auto& L = tileUpd[tl];
    std::stable_sort(L.begin(), L.end(), [&](int a, int b) { return est[a] < est[b]; });
    const bool hasSum = tl < nt && sumTask[tl] >= 0;
    const int base = hasSum ? 1 : 0;
    for (size_t q = 0; q < L.size(); ++q) {
      gen[L[q]].w0v = base + (int)q;
      if (q > 0) preds[L[q]].push_back(L[q - 1]);
      else if (hasSum) preds[L[q]].push_back(sumTask[tl]);
      if (tl >= nt && q == 0) gen[L[q]].flags |= 2;  // first update of a scratch tile overwrites
    }
    nupd[tl] = base + (int)L.size();
    if (tl < nt && finalTask[tl] >= 0) {
      if (!L.empty()) preds[finalTask[tl]].push_back(L.back());
      else if (hasSum) preds[finalTask[tl]].push_back(sumTask[tl]);
    }
  }
  for (int tl = 0; tl < nt; ++tl) {
    if (sumTask[tl] < 0) continue;
    BaTask& g = gen[sumTask[tl]];
    g.l0 = (int)P.sumList.size();
    std::sort(scratchOf[tl].begin(), scratchOf[tl].end());
    for (auto& e : scratchOf[tl]) {
      P.sumList.push_back({e.second, nupd[e.second]});
      preds[sumTask[tl]].push_back(tileUpd[e.second].back());
    }
    g.l1 = (int)P.sumList.size();
  }
  for (int t = 0; t < nFactorTasks; ++t) {
    BaTask& g = gen[t];
    if (g.type == BA_T_POTRF) {
      g.w0v = nupd[g.tC];
    } else if (g.type == BA_T_TRSM) {
      g.w0v = nupd[g.tC];
      g.w1v = nupd[g.w1i] + 1;
    } else if (g.type == BA_T_UPD) {
      g.w1v = nupd[g.tA] + 1;
      g.w2v = nupd[g.tB] + 1;
    }
  }
  for (int k = nb - 1; k >= 0; --k) {
    BaTask t = blank();
    t.type = BA_T_BWD;
    t.k = t.i = k;
    t.tC = T(k, k);
    t.tA = k;
    t.done = ntAll + k;
    t.w0i = T(k, k);
    t.w0v = nupd[T(k, k)] + 1;
    t.l0 = (int)P.bwdList.size();
    const int id = push(t, cBwd);
    preds[id].push_back(potrfTask[k]);
    // oldest solution first: x_i of the LARGEST i was produced first (BWD runs nb-1 .. 0), the smallest i
    // last -- the kernel polls per chunk of entries, so only the last chunk waits for the predecessor on
    // the chain while the others (and the tile loads of the last one) overlap with it
    for (auto it = strct[k].rbegin(); it != strct[k].rend(); ++it) {
      const int i = *it;
      P.bwdList.push_back({i, T(i, k), nupd[T(i, k)] + 1, 0});
      preds[id].push_back(bwdTask[i]);
    }
    gen[id].l1 = (int)P.bwdList.size();
    bwdTask[k] = id;
    P.flops += 2.0 * P.blkRows[k] * (double)P.blkRows[k] * (1.0 + (double)strct[k].size());
  }
  // ---- 4. critical-path-first list order ---------------------------------------------------
  const int ntask = (int)gen.size();
  std::vector<int> topo;
  {
    std::vector<int> indeg(ntask, 0);
    std::vector<std::vector<int>> succ(ntask);
    for (int t = 0; t < ntask; ++t)
      for (int p : preds[t]) {
        succ[p].push_back(t);
        ++indeg[t];
      }
    topo.reserve(ntask);
    for (int t = 0; t < ntask; ++t)
      if (!indeg[t]) topo.push_back(t);
    for (size_t h = 0; h < topo.size(); ++h)
      for (int s : succ[topo[h]])
        if (--indeg[s] == 0) topo.push_back(s);
    if ((int)topo.size() != ntask) {  // cannot happen (see the acyclicity argument in DESIGN.md)
      P.tasks.clear();
      P.nb = -1;
      return P;
    }
  }
  std::vector<double> bl(cost);
  std::vector<int> depthTasks(ntask, 1), topoPos(ntask);
  for (int h = ntask - 1; h >= 0; --h) {
    const int t = topo[h];
    topoPos[t] = h;
    for (int p : preds[t]) {
      if (cost[p] + bl[t] > bl[p]) bl[p] = cost[p] + bl[t];
      depthTasks[p] = std::max(depthTasks[p], depthTasks[t] + 1);
    }
  }
  std::vector<int> idx(topo);
  std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return bl[a] > bl[b]; });
  P.tasks.resize(ntask);
  for (int t = 0; t < ntask; ++t) P.tasks[t] = gen[idx[t]];
  for (int t = 0; t < ntask; ++t) {
    P.criticalPathCost = std::max(P.criticalPathCost, bl[t]);
    P.criticalPathTasks = std::max(P.criticalPathTasks, depthTasks[t]);
  }
  return P;
}

// ---- selected inversion Z = S^-1 on the factor's tile pattern (covariance of the BA, DESIGN.md 4.6) ----
// The Takahashi recurrences, walking the pivots from the last block to the first, with s = struct(k) =
// the blocks i > k that own a tile (i, k) of the factor (fill included):
//   Z_ik = -(sum_{j in s} Z_ij L_jk) L_kk^-1                  for every i in s
//   Z_kk = L_kk^-T (L_kk^-1 - sum_{i in s} L_ik^T Z_ik)
// Z_ij (i, j in s) is a tile of the pattern: the fill of pivot k joins every pair of s.  Every block of s is
// eliminated after k, so all those tiles are final when step k runs: one step per pivot, its off-diagonal
// tasks independent of each other, its diagonal task after them.  The order of the tasks of a step and of
// the operands of a task is fixed (ascending block), so the sums are deterministic.
struct BaSelTask {   // Z_ik (i > k), or Z_kk (i == k: the last task of its step)
  int k, i, tOut;    // tOut = tile index of (i, k), in the factor's layout
  int opBegin, opEnd;  // range in BaSelPlan::ops
};

struct BaSelOp {
  // off-diagonal task: Z_ij (tile tZ, read transposed when zT: the tile stores Z_ji) times L_jk (tile tL);
  // diagonal task: L_jk^T (tile tL) times Z_jk (tile tZ == tL)
  int tZ, zT, tL, j;
};

struct BaSelPlan {
  std::vector<int> stepBegin;  // step q (pivot k = nb - 1 - q): tasks [stepBegin[q], stepBegin[q + 1])
  std::vector<BaSelTask> tasks;
  std::vector<BaSelOp> ops;
};

inline BaSelPlan ba_make_selinv_plan(const BaPlan& P) {
  BaSelPlan S;
  const int nb = P.nb;
  auto T = [&](int i, int j) { return P.tileIdx[(size_t)i * nb + j]; };
  for (int k = nb - 1; k >= 0; --k) {
    S.stepBegin.push_back((int)S.tasks.size());
    std::vector<int> s;
    for (int i = k + 1; i < nb; ++i)
      if (T(i, k) >= 0) s.push_back(i);
    for (int i : s) {
      BaSelTask t{k, i, T(i, k), (int)S.ops.size(), 0};
      for (int j : s) S.ops.push_back({i >= j ? T(i, j) : T(j, i), i < j ? 1 : 0, T(j, k), j});
      t.opEnd = (int)S.ops.size();
      S.tasks.push_back(t);
    }
    BaSelTask d{k, k, T(k, k), (int)S.ops.size(), 0};
    for (int j : s) S.ops.push_back({T(j, k), 0, T(j, k), j});
    d.opEnd = (int)S.ops.size();
    S.tasks.push_back(d);
  }
  S.stepBegin.push_back((int)S.tasks.size());
  return S;
}

}  // namespace coslam
