// Test infrastructure (CPU): GlobalPoseGraph of coslam_b200/shim/SL_GlobalPoseEstimation.h compiled with
// COSL_POSEGRAPH_GENERAL against MOCKS of cosl_posegraph_spread_chains and cosl_posegraph_solve: the
// flattening of a merge-shaped graph, the scale-id -> column map of computeNewCameraTranslations4
// (slam/SL_GlobalPoseEstimation.cpp:383-403), the write-back of CamPoseEdge::s (:515-522), one ABI call
// for rotations + translations, chains still on the chain entry, and the refusals.
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "SL_GlobalPoseEstimation.h"

static int g_fail = 0, g_chainCalls = 0, g_solveCalls = 0, g_rc = 0;
static int g_expectScale = 0;
#define EXPECT(c)                                        \
  do {                                                   \
    if (!(c)) {                                          \
      std::printf("mock: expectation failed: %s\n", #c); \
      g_fail = 1;                                        \
    }                                                    \
  } while (0)

extern "C" {
const char* cosl_last_error(void) { return "mock failure"; }
int cosl_posegraph_spread_chains(int nChains, const int* off, const uint8_t*, const double*, const double*,
                                 const double*, const double*, double* newR, double* newt, int device) {
  ++g_chainCalls;
  EXPECT(nChains == 1 && device == 2);
  for (int g = 0; g < off[nChains]; ++g) {
    for (int i = 0; i < 9; ++i) newR[9 * g + i] = 500 + g;
    for (int i = 0; i < 3; ++i) newt[3 * g + i] = 600 + g;
  }
  return COSL_OK;
}
int cosl_posegraph_solve(int nNodes, const uint8_t* fixed, const double* R, const double* t, int nEdges,
                         const int* id1, const int* id2, const double* eR, const double* et, const int* scaleCol,
                         int nScale, double* newR, double* newt, double* scale, int device) {
  ++g_solveCalls;
  if (g_rc) return g_rc;
  EXPECT(device == 2 && nScale == g_expectScale);
  for (int k = 0; k < nNodes; ++k) {
    EXPECT(fixed[k] == (k < 2 ? 1 : 0));
    EXPECT(R[9 * k] == 10 + k && t[3 * k + 2] == -k);
  }
  for (int e = 0; e < nEdges; ++e) {
    EXPECT(eR[9 * e + 4] == 100 + e && et[3 * e + 1] == 200 + e);
    EXPECT(id1[e] >= 0 && id1[e] < nNodes && id2[e] >= 0 && id2[e] < nNodes);
  }
  if (g_expectScale == 2) {  // the constraint edges 7 (id 3) and 8 (id 1), 9 (id 3): ids {1, 3} -> columns {0, 1}
    for (int e = 0; e < 7; ++e) EXPECT(scaleCol[e] == -1);
    EXPECT(scaleCol[7] == 1 && scaleCol[8] == 0 && scaleCol[9] == 1);
    EXPECT(id1[8] == 3 && id2[8] == 4);
  } else {
    for (int e = 0; e < nEdges; ++e) EXPECT(scaleCol[e] == -1);
  }
  for (int g = 0; g < nNodes; ++g) {
    for (int i = 0; i < 9; ++i) newR[9 * g + i] = 7000 + g + 0.01 * i;
    for (int i = 0; i < 3; ++i) newt[3 * g + i] = 8000 + g + 0.01 * i;
  }
  for (int c = 0; c < nScale; ++c) scale[c] = 11 + 2 * c;
  return COSL_OK;
}
}

// 3 key frames x 2 cameras (node 2k + c), the first key frame fixed
static void merge_graph(GlobalPoseGraph& g, bool constraints) {
  g.clear();
  g.device = 2;
  g.reserve(6, 18);
  for (int k = 0; k < 6; ++k) {
    double R[9] = {0}, t[3] = {0};
    R[0] = 10 + k;
    t[2] = -k;
    CamPoseNode* nd = g.newNode();
    nd->set(k / 2, k % 2, R, t);
    nd->fixed = k < 2;
  }
  const int ends[10][2] = {{0, 1}, {2, 3}, {0, 2}, {1, 3}, {4, 5}, {2, 4}, {3, 5}, {5, 2}, {3, 4}, {4, 3}};
  const int sid[10] = {-1, -1, -1, -1, -1, -1, -1, 3, 1, 3};
  const int n = constraints ? 10 : 7;
  for (int e = 0; e < n; ++e) {
    double R[9] = {0}, t[3] = {0};
    R[4] = 100 + e;
    t[1] = 200 + e;
    CamPoseEdge* ed = g.addEdge();
    if (sid[e] < 0) {
      ed->set(ends[e][0], ends[e][1], R, t);
    } else {
      ed->set(ends[e][0], ends[e][1], R, t, sid[e]);
      ed->uncertainScale = true;
      ed->constraint = true;
      g.nConstraintEdge++;
    }
  }
}

int main() {
  GlobalPoseGraph g;
  merge_graph(g, true);
  g_expectScale = 2;
  g.computeNewCameraRotations();
  EXPECT(g_solveCalls == 1 && g_chainCalls == 0);
  EXPECT(g.poseNodes[3].newR[2] == 7003.02 && g.poseNodes[3].newt[2] == -3.0);  // newt = t after the rotations
  g.computeNewCameraTranslations4();
  EXPECT(g_solveCalls == 1);  // both halves from ONE call
  EXPECT(g.poseNodes[3].newR[2] == 7003.02 && g.poseNodes[3].newt[1] == 8003.01);
  EXPECT(g.poseNodes[1].newR[0] == 11.0);  // fixed: newR = R (:505-513; newt comes from the ABI)
  EXPECT(g.poseEdges[7].s == 13 && g.poseEdges[8].s == 11 && g.poseEdges[9].s == 13);
  for (int e = 0; e < 7; ++e) EXPECT(g.poseEdges[e].s == 0);
  g.computeNewCameraTranslations4();  // alone: a fresh solve
  EXPECT(g_solveCalls == 2);
  // the per-edge-scale form is refused
  bool threw = false;
  try { g.computeNewCameraTranslations(); } catch (const std::runtime_error&) { threw = true; }
  EXPECT(threw && g_solveCalls == 2);
  // an uncertain edge whose scale id no constraint edge carries (the reference aliases column -1)
  g.poseEdges[9].constraint = false;
  g.poseEdges[9].scaleId = 5;
  threw = false;
  try { g.computeNewCameraRotations(); } catch (const std::runtime_error&) { threw = true; }
  EXPECT(threw && g_solveCalls == 2);
  // a general graph without uncertain edges: rotations + translations = one solve call, no scales
  merge_graph(g, false);
  g_expectScale = 0;
  g.computeNewCameraRotations();
  g.computeNewCameraTranslations();
  EXPECT(g_solveCalls == 3 && g_chainCalls == 0);
  EXPECT(g.poseNodes[4].newt[0] == 8004.0);
  // chains still take the chain entry
  GlobalPoseGraph c;
  c.device = 2;
  c.reserve(5, 4);
  for (int k = 0; k < 5; ++k) {
    double R[9] = {0}, t[3] = {0};
    c.newNode()->set(k, 0, R, t);
  }
  c.poseNodes[0].fixed = true;
  for (int k = 0; k < 4; ++k) {
    double R[9] = {0}, t[3] = {0};
    c.addEdge()->set(k, k + 1, R, t);
  }
  c.computeNewCameraRotations();
  c.computeNewCameraTranslations();
  EXPECT(g_chainCalls == 1 && g_solveCalls == 3);
  EXPECT(c.poseNodes[2].newR[0] == 502 && c.poseNodes[2].newt[0] == 602);
  // ABI failure -> exception carrying cosl_last_error()
  g_rc = COSL_E_INVALID;
  threw = false;
  try { g.computeNewCameraRotations(); } catch (const std::runtime_error& e) { threw = std::strstr(e.what(), "mock failure") != 0; }
  EXPECT(threw);
  if (!g_fail) std::printf("MOCK_POSEGRAPH_GENERAL_OK\n");
  return g_fail;
}
