// Test infrastructure (GPU): a merge-shaped key-frame graph through coslam_b200/shim/SL_GlobalPoseEstimation.h
// compiled with COSL_POSEGRAPH_GENERAL, built and solved the way MergeCameraGroup does it
// (reference app/SL_MergeCameraGroup.cpp:907-1035, :1083-1086).  Input: the binary graph written by
// tests/test_gpu_posegraph_general.py; output: "ok" and newR, newt of every node, s of every edge.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "SL_GlobalPoseEstimation.h"

template <class T>
static bool rd(std::FILE* f, std::vector<T>& v, size_t n) {
  v.resize(n);
  return n == 0 || std::fread(v.data(), sizeof(T), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<int> hdr, fixed, id1, id2, sid;
  std::vector<double> R, t, eR, et;
  bool ok = rd(f, hdr, 2);
  const int n = ok ? hdr[0] : 0, ne = ok ? hdr[1] : 0;
  ok = ok && rd(f, fixed, n) && rd(f, R, 9 * (size_t)n) && rd(f, t, 3 * (size_t)n) && rd(f, id1, ne) &&
       rd(f, id2, ne) && rd(f, eR, 9 * (size_t)ne) && rd(f, et, 3 * (size_t)ne) && rd(f, sid, ne);
  std::fclose(f);
  if (!ok) return 2;
  GlobalPoseGraph keyGraph;
  keyGraph.clear();
  keyGraph.reserve(n, ne);
  keyGraph.nFixedNode = 0;
  for (int k = 0; k < n; ++k) {
    CamPoseNode* pNode = keyGraph.newNode();
    pNode->set(k, 0, &R[9 * (size_t)k], &t[3 * (size_t)k]);
    pNode->fixed = fixed[k] != 0;
    if (pNode->fixed) keyGraph.nFixedNode++;
  }
  keyGraph.nConstraintEdge = 0;
  for (int e = 0; e < ne; ++e) {
    CamPoseEdge* pEdge = keyGraph.addEdge();
    if (sid[e] < 0) {
      pEdge->set(id1[e], id2[e], &eR[9 * (size_t)e], &et[3 * (size_t)e]);
    } else {
      pEdge->set(id1[e], id2[e], &eR[9 * (size_t)e], &et[3 * (size_t)e], sid[e]);
      pEdge->uncertainScale = true;
      pEdge->constraint = true;
      keyGraph.poseNodes[id1[e]].constraint = true;
      keyGraph.poseNodes[id2[e]].constraint = true;
      keyGraph.nConstraintEdge++;
    }
  }
  try {
    keyGraph.computeNewCameraRotations();
    keyGraph.computeNewCameraTranslations4();
  } catch (const std::runtime_error& e) {
    std::printf("error %s\n", e.what());
    return 1;
  }
  std::printf("ok");
  for (int k = 0; k < n; ++k)
    for (int i = 0; i < 9; ++i) std::printf(" %.17g", keyGraph.poseNodes[k].newR[i]);
  for (int k = 0; k < n; ++k)
    for (int i = 0; i < 3; ++i) std::printf(" %.17g", keyGraph.poseNodes[k].newt[i]);
  for (int e = 0; e < ne; ++e) std::printf(" %.17g", keyGraph.poseEdges[e].s);
  std::printf("\n");
  return 0;
}
