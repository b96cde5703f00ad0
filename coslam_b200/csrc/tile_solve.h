// tile_solve.h -- set-up and launch of the block-sparse SPD solve of ba_tile.cuh (plain C++).
//
// ba_tile.cuh defines its kernels with external linkage, so it is included by ba.cu alone.  Every caller of
// the solve (the BA solver's LM trial and covariance stage, the general pose graph of posegraph.cu, the debug
// entry points) derives the launch, the device image of the plan's lists and the kernel arguments from a
// BaPlan through the functions below.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "ba_plan.h"

namespace coslam {

// Arguments of ba_tile_solve / ba_tile_two.
struct BaTileDev {
  double* rhs;    // [nb*64]
  double* tiles;  // [nTiles + nScratch][4096]  (scratch tiles: see ba_plan.h)
  double* rhsS;   // [nScratch*64] rhs parts that travel with the scratch tiles of diagonal tiles
  double* Linv;   // [nb][4096]
  double* y;      // [nb*64]
  double* x;      // [nb*64]
  int* cnt;       // [nCounters + 2 + nTasks]: counters, the two task tickets of the CTA roles, claim flags
  const BaTask* tasks;
  const BaBwdEntry* bwd;
  const BaSumEntry* sum;
  const int* blkRows;
  int nTasks, nb, nTiles, nCounters;
  int nA;        // tasks [0, nA) = POTRF / BACKWARD (specialist CTAs), [nA, nTasks) = TRSM / UPDATE / SUM
  int nSpecial;  // CTAs [0, nSpecial) serve the first list: code working sets stay inside the I-cache
  int xdoneBase;  // counter index of "x_0 done" (= nTiles + nScratch)
  double* sc;
  int scFail;
  unsigned long long* trace;  // optional [nTasks][8]: sm id, ns at ticket / ready / done, 4 phase stamps
};

// How the solve of one plan is launched.
struct TileLaunch {
  // The plan's tasks in the order the persistent kernel takes them: POTRF / BWD first (served by the
  // specialist CTAs), then TRSM / UPD / SUM, with the hot successors of every POTRF filled in.  nA: the
  // number of tasks of the first list.
  std::vector<BaTask> order;
  int nA = 0;
  // One or two blocks with their diagonal tiles: one resident CTA (ba_tile_two) on tiles t00, t10, t11.
  bool two = false;
  int t00 = -1, t10 = -1, t11 = -1;
  // The persistent kernel's grid (never more CTAs than can be co-resident: the tickets spin) and its
  // specialist CTAs; set by tile_launch_device.
  int grid = 0, nSpecial = 0;
};

// The host half of the launch: task order and the small-solve choice.
TileLaunch tile_launch_plan(const BaPlan& P);

// The device half on the current device: grid and nSpecial.  The first call on a device also sets the shared
// memory limits of the solve and selected-inversion kernels there.
int tile_launch_device(TileLaunch& L);

// The plan's read-only lists as one block of `bytes` bytes in 256-byte-aligned sections: tasks in ticket order,
// BACKWARD and SUM lists, blkRows, blkCam0, order, the tile -> diagonal block map and its inverse.  tile_image
// lays it out, tile_image_write writes it into a host buffer (the caller's staging buffer: no extra copy).
struct TileImage {
  size_t bytes = 0, tasks = 0, bwd = 0, sum = 0, blkRows = 0, blkCam0 = 0, order = 0, diagBlk = 0, diagTile = 0;
};
TileImage tile_image(const BaPlan& P, const TileLaunch& L);
void tile_image_write(const BaPlan& P, const TileLaunch& L, const TileImage& I, unsigned char* dst);

// The lists of an image uploaded to `base`.
struct TileLists {
  const BaTask* tasks;
  const BaBwdEntry* bwd;
  const BaSumEntry* sum;
  const int* blkRows;
  const int* blkCam0;
  const int* order;
  const int* diagBlk;   // [max(1, nTiles)]: block of a diagonal tile, -1 for the others
  const int* diagTile;  // [max(1, nb)]: tile of block k's diagonal
};
TileLists tile_lists(const TileImage& I, const void* base);

// The arguments of the solve with the counts of the plan and the launch and the lists; the caller sets the
// work buffers (rhs, tiles, rhsS, Linv, y, x, cnt) and the failure flag (sc, scFail: set to 1 on a
// non-positive or out-of-range pivot, never cleared here).
BaTileDev tile_dev(const BaPlan& P, const TileLaunch& L, const TileLists& lists);

// Enqueues the solve of the assembled system on `s`: x = S^-1 rhs, block padded in the plan's order.  The
// counters and tickets (cnt) must be zero.
int tile_solve_enqueue(const TileLaunch& L, const BaTileDev& td, cudaStream_t s);

}  // namespace coslam
