/* TEST INFRASTRUCTURE.  A second C entry into the UNMODIFIED reference file slam/SL_GlobalPoseEstimation.cpp,
 * linked with the stand-ins of primitives_pg.cpp into oracle/_ref/libposegraph_merge_ref.so
 * (oracle/Makefile.pg_general): the camera-group merge's key-frame solve,
 * GlobalPoseGraph::computeNewCameraRotations (:52-218) + ::computeNewCameraTranslations4 (:361-525).
 * The sparse least squares of that path is the stand-in sparseSolveLin (dense Householder QR). */
#include <cstring>

#include "SL_GlobalPoseEstimation.h"

/* C entry: builds the graph the way MergeCameraGroup::_constructGraphForKeyFrms does
 * (app/SL_MergeCameraGroup.cpp:907-1035) -- an edge with scaleId[e] >= 0 is a merge constraint: set with
 * that scale id, uncertainScale = constraint = true, its nodes marked constraint, nConstraintEdge counted
 * -- and runs recomputeKeyCamPoses' two solves (:1083-1086).  s[e] = CamPoseEdge::s afterwards. */
extern "C" void ref_posegraph_merge(int nNodes, const int* fixed, const double* R, const double* t, int nEdges,
                                    const int* id1, const int* id2, const double* eR, const double* et,
                                    const int* scaleId, double* newR, double* newt, double* s) {
  GlobalPoseGraph g;
  g.reserve(nNodes, nEdges > 0 ? nEdges : 1);
  g.nFixedNode = 0;
  for (int k = 0; k < nNodes; ++k) {
    CamPoseNode* nd = g.newNode();
    nd->set(k, 0, R + 9 * k, t + 3 * k);
    nd->fixed = fixed[k] != 0;
    if (nd->fixed) g.nFixedNode++;
  }
  g.nConstraintEdge = 0;
  for (int e = 0; e < nEdges; ++e) {
    CamPoseEdge* ed = g.addEdge();
    if (scaleId[e] < 0) {
      ed->set(id1[e], id2[e], eR + 9 * e, et + 3 * e);
    } else {
      ed->set(id1[e], id2[e], eR + 9 * e, et + 3 * e, scaleId[e]);
      ed->uncertainScale = true;
      ed->constraint = true;
      g.poseNodes[id1[e]].constraint = true;
      g.poseNodes[id2[e]].constraint = true;
      g.nConstraintEdge++;
    }
  }
  g.computeNewCameraRotations();
  g.computeNewCameraTranslations4();
  for (int k = 0; k < nNodes; ++k) {
    std::memcpy(newR + 9 * k, g.poseNodes[k].newR, 72);
    std::memcpy(newt + 3 * k, g.poseNodes[k].newt, 24);
  }
  for (int e = 0; e < nEdges; ++e) s[e] = g.poseEdges[e].s;
}
