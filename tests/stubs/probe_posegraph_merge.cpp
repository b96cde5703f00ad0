// Test infrastructure: written against the reference's slam/SL_GlobalPoseEstimation.h and compiled with
// coslam_b200/shim/SL_GlobalPoseEstimation.h in its place and COSL_POSEGRAPH_GENERAL defined
// (tests/test_posegraph_general.py).  The body follows the calls of MergeCameraGroup::
// _constructGraphForKeyFrms, ::recomputeKeyCamPoses and ::recomputeAllCameraPoses (reference
// app/SL_MergeCameraGroup.cpp:907-1035, :1083-1120), with the key-frame containers reduced to arrays.
#include <cassert>  // the reference header gets it through LibVisualSLAM's math/SL_Matrix.h
#include <cstring>
#include <vector>

#include "slam/SL_GlobalPoseEstimation.h"

struct ProbeMerge {
  int m_nMergeInfo;
  GlobalPoseGraph keyGraph;
  GlobalPoseGraph camGraphs[4];
  std::vector<double*> m_pKeyPoses;

  void _constructGraphForKeyFrms(int nKey, int nCam, double* R, double* t, const int* mf, const double* mR,
                                 const double* mt, GlobalPoseGraph& graph) {
    graph.clear();
    int nTotalNode = nKey * nCam;
    graph.reserve(nTotalNode, nTotalNode * 3);
    m_pKeyPoses.clear();
    m_pKeyPoses.reserve(nTotalNode);
    graph.nFixedNode = 0;
    for (int kf = 0; kf < nKey; ++kf)
      for (int c = 0; c < nCam; ++c) {
        CamPoseNode* pNode = graph.newNode();
        pNode->set(kf, c, R + 9 * pNode->id, t + 3 * pNode->id);
        pNode->fixed = kf == 0 ? true : false;
        m_pKeyPoses.push_back(R + 9 * pNode->id);
        if (pNode->fixed) graph.nFixedNode++;
      }
    double eR[9], et[3];
    for (int kf = 0; kf < nKey; ++kf) {
      size_t i = 1;
      for (; i < (size_t)nCam; i++) {
        CamPoseEdge* pEdge = graph.addEdge();
        pEdge->set(kf * nCam + (int)i - 1, kf * nCam + (int)i, eR, et);
      }
      if (nCam > 2) {
        CamPoseEdge* pEdge = graph.addEdge();
        pEdge->set(kf * nCam + (int)i - 1, kf * nCam, eR, et);
      }
      if (kf > 0)
        for (int c = 0; c < nCam; ++c) {
          CamPoseEdge* pEdge = graph.addEdge();
          pEdge->set((kf - 1) * nCam + c, kf * nCam + c, eR, et);
        }
    }
    graph.nConstraintEdge = 0;
    for (int i = 0; i < m_nMergeInfo; i++) {
      int nodeId1 = mf[2 * i], nodeId2 = mf[2 * i + 1];
      CamPoseEdge* pEdge = graph.addEdge();
      pEdge->set(nodeId1, nodeId2, mR + 9 * i, mt + 3 * i, 0);
      pEdge->uncertainScale = true;
      pEdge->constraint = true;
      graph.poseNodes[nodeId1].constraint = true;
      graph.poseNodes[nodeId2].constraint = true;
      graph.nConstraintEdge++;
    }
  }
  void recomputeKeyCamPoses() {
    keyGraph.computeNewCameraRotations();
    keyGraph.computeNewCameraTranslations4();
    for (int i = 0; i < keyGraph.nNodes; i++) {
      double* cam = m_pKeyPoses[i];
      memcpy(cam, keyGraph.poseNodes[i].newR, sizeof(double) * 9);
      memcpy(cam + 9, keyGraph.poseNodes[i].newt, sizeof(double) * 3);
      int c = keyGraph.poseNodes[i].camId;
      memcpy(camGraphs[c].poseNodes[0].R, cam, sizeof(double) * 9);
      memcpy(camGraphs[c].poseNodes[0].t, cam + 9, sizeof(double) * 3);
    }
  }
  void recomputeAllCameraPoses() {
    for (int c = 0; c < 4; c++) {
      camGraphs[c].computeNewCameraRotations();
      camGraphs[c].computeNewCameraTranslations();
    }
  }
  double scale() const { return keyGraph.poseEdges[keyGraph.nEdges - 1].s; }
};
