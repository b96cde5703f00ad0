// tile_solve.h -- the block-sparse SPD solve of ba_tile.cuh for callers outside ba.cu (plain C++).
//
// ba_tile.cuh defines its kernels with external linkage, so it is included by ba.cu alone; other
// translation units that own an SPD system with the tile layout of ba_plan.h (the general pose graph
// of posegraph.cu) reach the same kernels through these two functions.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "ba_plan.h"

namespace coslam {

// The plan's tasks in the order the persistent kernel takes them: POTRF / BWD first (served by the
// specialist CTAs), then TRSM / UPD / SUM, with the hot successors of every POTRF filled in.
// Returns the number of tasks of the first list.
int tile_task_order(const BaPlan& P, std::vector<BaTask>& order);

// Device buffers of one solve; sizes as ba_tile.cuh documents them (rhs, y, x: nb*64; tiles:
// (nTiles + nScratch)*4096; rhsS: max(1, nScratch)*64; Linv: nb*4096; cnt: nCounters + 2 + nTasks).
struct TileSolveBufs {
  double* rhs;
  double* tiles;
  double* rhsS;
  double* Linv;
  double* y;
  double* x;
  int* cnt;
  const BaTask* tasks;  // tile_task_order's list
  const BaBwdEntry* bwd;
  const BaSumEntry* sum;
  const int* blkRows;
  double* fail;  // set to 1 on a non-positive or out-of-range pivot; never cleared here
};

// Enqueues the solve of the assembled system on `s`: x = S^-1 rhs, block padded in the plan's
// order.  The counters and tickets (cnt) must be zero.  One CTA for one or two blocks (ba_tile_two),
// the persistent dataflow kernel (ba_tile_solve) otherwise.  gridOut (optional): CTAs launched.
int tile_solve_launch(const BaPlan& P, int nA, const TileSolveBufs& b, int device, cudaStream_t s,
                      int* gridOut = nullptr);

}  // namespace coslam
