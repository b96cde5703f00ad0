// Drop-in for slam/SL_GlobalPoseEstimation.h of danping/CoSLAM: CamPoseNode (:13-41), CamPoseEdge
// (:42-70) and the part of GlobalPoseGraph (:72-117) that the post-BA path uses --
// RobustBundleRTS::constructCameraGraphs / updateNonKeyCameraPoses (app/SL_CoSLAMRobustBA.cpp:182-250)
// compile unchanged.  computeNewCameraRotations() + computeNewCameraTranslations() forward to ONE
// cosl_posegraph_spread_chains call (the kernel solves both systems in the same pass); the result of
// the translation half is cached until the graph is touched again through clear()/newNode()/addEdge().
//
// Supported graphs: what constructCameraGraphs builds -- edge e runs from node e to node e+1, no
// uncertain-scale edges.  Anything else throws std::runtime_error (the constrained variants
// computeNewCamera*2/3/4 and save/load are not on the post-BA path and are not provided).
//
// With COSL_POSEGRAPH_GENERAL defined (for EVERY translation unit of the program: the class layout and
// its inline methods differ, so mixing breaks the one-definition rule) the header also serves
// MergeCameraGroup (app/SL_MergeCameraGroup.cpp:907-1102): computeNewCameraRotations /
// computeNewCameraTranslations accept any edge set without uncertain-scale edges, and
// computeNewCameraTranslations4() solves the shared-scale translations.  Chain graphs without
// uncertain edges still go to cosl_posegraph_spread_chains (the same bits as without the definition);
// every other graph goes to cosl_posegraph_solve.  A rotations call followed by a translations call is
// one ABI call either way.
#ifndef SL_GLOBALPOSEESTIMATION_H_
#define SL_GLOBALPOSEESTIMATION_H_
#include <cassert>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "coslam_b200.h"

class CamPoseNode {
public:
	int id;
	int frame;
	int camId;
	bool fixed;
	double R[9];
	double t[3];
	double newR[9];
	double newt[3];
	bool constraint;
public:
	CamPoseNode() :
			id(-1), frame(-1), camId(-1), fixed(false), constraint(false) {
	}
	void set(const double RMat[9], const double tMat[3]) {
		std::memcpy(R, RMat, sizeof(double) * 9);
		std::memcpy(newR, RMat, sizeof(double) * 9);
		std::memcpy(t, tMat, sizeof(double) * 3);
		std::memcpy(newt, tMat, sizeof(double) * 3);
	}
	void set(int f, int cameraId, const double RMat[9], const double tMat[3]) {
		frame = f;
		camId = cameraId;
		set(RMat, tMat);
	}
};

class CamPoseEdge {
public:
	int id1, id2;
	bool constraint;
	bool uncertainScale;
	double R[9];
	double t[3];
	double s;
	int scaleId;
public:
	CamPoseEdge() :
			id1(-1), id2(-1), constraint(0), uncertainScale(false), s(0), scaleId(-1) {
	}
	void set(int nodeId1, int nodeId2, const double RMat[9], const double tMat[3]) {
		id1 = nodeId1;
		id2 = nodeId2;
		std::memcpy(R, RMat, sizeof(double) * 9);
		std::memcpy(t, tMat, sizeof(double) * 3);
		s = 0;
	}
	void set(int nodeId1, int nodeId2, const double RMat[9], const double tMat[3], int sId) {
		set(nodeId1, nodeId2, RMat, tMat);
		scaleId = sId;
	}
};

class GlobalPoseGraph {
public:
	int nNodes;
	CamPoseNode* poseNodes;
	int nEdges;
	CamPoseEdge* poseEdges;
	int nFixedNode;
	int nConstraintEdge;
	int nMaxNodes;
	int nMaxEdges;
	int device;  // CUDA device of the solve (extension; default 0)
public:
	GlobalPoseGraph() :
			nNodes(0), poseNodes(0), nEdges(0), poseEdges(0), nFixedNode(0), nConstraintEdge(0), nMaxNodes(0),
			nMaxEdges(0), device(0), m_haveT(false) {
	}
	virtual ~GlobalPoseGraph() {
		clear();
	}
	void reserve(int numMaxNodes, int numMaxEdges) {
		clear();
		nMaxNodes = numMaxNodes;
		nMaxEdges = numMaxEdges;
		poseNodes = new CamPoseNode[numMaxNodes > 0 ? numMaxNodes : 1];
		poseEdges = new CamPoseEdge[numMaxEdges > 0 ? numMaxEdges : 1];
	}
	void clear() {
		delete[] poseNodes;
		delete[] poseEdges;
		poseNodes = 0;
		poseEdges = 0;
		nNodes = nEdges = nMaxNodes = nMaxEdges = 0;
		nFixedNode = nConstraintEdge = 0;
		m_haveT = false;
	}
	CamPoseNode* newNode() {
		assert(nNodes < nMaxNodes);
		m_haveT = false;
		poseNodes[nNodes].id = nNodes;
		return &poseNodes[nNodes++];
	}
	CamPoseEdge* addEdge() {
		assert(nEdges < nMaxEdges);
		m_haveT = false;
		return &poseEdges[nEdges++];
	}

	// slam/SL_GlobalPoseEstimation.cpp:52-218: newR = spread rotations, newt = t
	void computeNewCameraRotations() {
		solve();
		for (int k = 0; k < nNodes; ++k) {
			std::memcpy(poseNodes[k].newR, &m_newR[9 * (size_t) k], sizeof(double) * 9);
			std::memcpy(poseNodes[k].newt, poseNodes[k].t, sizeof(double) * 3);
		}
		m_haveT = true;
	}
	// slam/SL_GlobalPoseEstimation.cpp:220-359: newt = spread translations (newR of free nodes untouched,
	// fixed nodes get copies of R, t as at :339-343)
	void computeNewCameraTranslations() {
#ifdef COSL_POSEGRAPH_GENERAL
		for (int e = 0; e < nEdges; ++e)
			if (poseEdges[e].uncertainScale)
				throw std::runtime_error("GlobalPoseGraph (coslam_b200): computeNewCameraTranslations with uncertain-scale edges is not supported (use computeNewCameraTranslations4)");
#endif
		if (!m_haveT)
			solve();
		for (int k = 0; k < nNodes; ++k) {
			if (poseNodes[k].fixed)
				std::memcpy(poseNodes[k].newR, poseNodes[k].R, sizeof(double) * 9);
			std::memcpy(poseNodes[k].newt, &m_newt[3 * (size_t) k], sizeof(double) * 3);
		}
		m_haveT = false;
	}
#ifdef COSL_POSEGRAPH_GENERAL
	// slam/SL_GlobalPoseEstimation.cpp:361-525: newt = translations with one unknown scale per scale id of
	// the constraint edges (:383-403); fixed nodes get copies of R, t (:505-513); CamPoseEdge::s of every
	// uncertain-scale edge = its solved scale (:515-522)
	void computeNewCameraTranslations4() {
		if (!m_haveT)
			solve();
		for (int k = 0; k < nNodes; ++k) {
			if (poseNodes[k].fixed)
				std::memcpy(poseNodes[k].newR, poseNodes[k].R, sizeof(double) * 9);
			std::memcpy(poseNodes[k].newt, &m_newt[3 * (size_t) k], sizeof(double) * 3);
		}
		for (int e = 0; e < nEdges; ++e)
			if (poseEdges[e].uncertainScale && poseEdges[e].scaleId >= 0)
				poseEdges[e].s = m_scale[m_scaleCol[e]];
		m_haveT = false;
	}
#endif
private:
	std::vector<double> m_newR, m_newt;
#ifdef COSL_POSEGRAPH_GENERAL
	std::vector<double> m_scale;
	std::vector<int> m_scaleCol;
#endif
	bool m_haveT;
	GlobalPoseGraph(const GlobalPoseGraph&);
	GlobalPoseGraph& operator=(const GlobalPoseGraph&);

	void solve() {
		const size_t n = (size_t) nNodes;
		m_newR.assign(9 * n, 0.0);
		m_newt.assign(3 * n, 0.0);
		if (nNodes == 0)
			return;
#ifdef COSL_POSEGRAPH_GENERAL
		bool chain = nEdges == nNodes - 1;
		for (int e = 0; chain && e < nEdges; ++e)
			chain = poseEdges[e].id1 == e && poseEdges[e].id2 == e + 1 && !poseEdges[e].uncertainScale;
		if (!chain) {
			solveGeneral();
			return;
		}
#endif
		if (nEdges != nNodes - 1)
			throw std::runtime_error("GlobalPoseGraph (coslam_b200): only chain graphs are supported (nEdges != nNodes-1)");
		std::vector<double> R(9 * n), t(3 * n), eR(9 * n, 0.0), et(3 * n, 0.0);
		std::vector<uint8_t> fixed(n);
		for (int k = 0; k < nNodes; ++k) {
			std::memcpy(&R[9 * (size_t) k], poseNodes[k].R, sizeof(double) * 9);
			std::memcpy(&t[3 * (size_t) k], poseNodes[k].t, sizeof(double) * 3);
			fixed[k] = poseNodes[k].fixed ? 1 : 0;
		}
		for (int e = 0; e < nEdges; ++e) {
			const CamPoseEdge& ed = poseEdges[e];
			if (ed.id1 != e || ed.id2 != e + 1)
				throw std::runtime_error("GlobalPoseGraph (coslam_b200): only chain graphs are supported (edge e must join node e to node e+1)");
			if (ed.uncertainScale)
				throw std::runtime_error("GlobalPoseGraph (coslam_b200): uncertain-scale edges are not supported");
			std::memcpy(&eR[9 * (size_t) e], ed.R, sizeof(double) * 9);
			std::memcpy(&et[3 * (size_t) e], ed.t, sizeof(double) * 3);
		}
		const int off[2] = { 0, nNodes };
		const int rc = cosl_posegraph_spread_chains(1, off, fixed.data(), R.data(), t.data(), eR.data(), et.data(),
				m_newR.data(), m_newt.data(), device);
		if (rc != COSL_OK)
			throw std::runtime_error(std::string("GlobalPoseGraph (coslam_b200): ") + cosl_last_error());
	}
#ifdef COSL_POSEGRAPH_GENERAL
	// any edge set: scale ids -> columns as :383-403 (the distinct ids of the constraint edges, in
	// increasing order); an uncertain edge whose id no constraint edge carries is refused (the reference
	// reads column -1 there, which aliases the last translation unknown)
	void solveGeneral() {
		const size_t n = (size_t) nNodes, ne = (size_t) nEdges;
		std::vector<int> colOfId(ne, -1), id1(ne), id2(ne);
		for (int e = 0; e < nEdges; ++e)
			if (poseEdges[e].constraint) {
				const int sId = poseEdges[e].scaleId;
				if (sId < 0 || sId >= nEdges)
					throw std::runtime_error("GlobalPoseGraph (coslam_b200): constraint edge with a scale id outside [0, nEdges)");
				colOfId[sId] = 0;
			}
		int nScale = 0;
		for (int k = 0; k < nEdges; ++k)
			if (colOfId[k] >= 0)
				colOfId[k] = nScale++;
		m_scaleCol.assign(ne, -1);
		std::vector<double> R(9 * n), t(3 * n), eR(9 * ne), et(3 * ne);
		std::vector<uint8_t> fixed(n);
		for (int k = 0; k < nNodes; ++k) {
			std::memcpy(&R[9 * (size_t) k], poseNodes[k].R, sizeof(double) * 9);
			std::memcpy(&t[3 * (size_t) k], poseNodes[k].t, sizeof(double) * 3);
			fixed[k] = poseNodes[k].fixed ? 1 : 0;
		}
		for (int e = 0; e < nEdges; ++e) {
			const CamPoseEdge& ed = poseEdges[e];
			id1[e] = ed.id1;
			id2[e] = ed.id2;
			std::memcpy(&eR[9 * (size_t) e], ed.R, sizeof(double) * 9);
			std::memcpy(&et[3 * (size_t) e], ed.t, sizeof(double) * 3);
			if (ed.uncertainScale) {
				const int c = (ed.scaleId >= 0 && ed.scaleId < nEdges) ? colOfId[ed.scaleId] : -1;
				if (c < 0)
					throw std::runtime_error("GlobalPoseGraph (coslam_b200): an uncertain-scale edge has a scale id that no constraint edge carries");
				m_scaleCol[e] = c;
			}
		}
		m_scale.assign(nScale > 0 ? nScale : 1, 0.0);
		const int rc = cosl_posegraph_solve(nNodes, fixed.data(), R.data(), t.data(), nEdges, id1.data(), id2.data(),
				eR.data(), et.data(), m_scaleCol.data(), nScale, m_newR.data(), m_newt.data(), m_scale.data(), device);
		if (rc != COSL_OK)
			throw std::runtime_error(std::string("GlobalPoseGraph (coslam_b200): ") + cosl_last_error());
	}
#endif
};

// All cameras' graphs in ONE launch (what updateNonKeyCameraPoses' loop over cameras becomes when the
// caller is free to batch): fills newR/newt of every node of graphs[0..nGraphs).
inline void computeNewCameraPosesBatch(GlobalPoseGraph* graphs, int nGraphs, int device = 0) {
	std::vector<int> off(nGraphs + 1, 0);
	for (int c = 0; c < nGraphs; ++c)
		off[c + 1] = off[c] + graphs[c].nNodes;
	const size_t n = (size_t) off[nGraphs];
	if (n == 0)
		return;
	std::vector<double> R(9 * n), t(3 * n), eR(9 * n, 0.0), et(3 * n, 0.0), nR(9 * n), nt(3 * n);
	std::vector<uint8_t> fixed(n);
	for (int c = 0; c < nGraphs; ++c) {
		const GlobalPoseGraph& g = graphs[c];
		if (g.nNodes > 0 && g.nEdges != g.nNodes - 1)
			throw std::runtime_error("computeNewCameraPosesBatch: only chain graphs are supported");
		for (int k = 0; k < g.nNodes; ++k) {
			const size_t i = (size_t) off[c] + k;
			std::memcpy(&R[9 * i], g.poseNodes[k].R, sizeof(double) * 9);
			std::memcpy(&t[3 * i], g.poseNodes[k].t, sizeof(double) * 3);
			fixed[i] = g.poseNodes[k].fixed ? 1 : 0;
		}
		for (int e = 0; e < g.nEdges; ++e) {
			const CamPoseEdge& ed = g.poseEdges[e];
			if (ed.id1 != e || ed.id2 != e + 1 || ed.uncertainScale)
				throw std::runtime_error("computeNewCameraPosesBatch: only chain graphs without uncertain scale are supported");
			std::memcpy(&eR[9 * ((size_t) off[c] + e)], ed.R, sizeof(double) * 9);
			std::memcpy(&et[3 * ((size_t) off[c] + e)], ed.t, sizeof(double) * 3);
		}
	}
	const int rc = cosl_posegraph_spread_chains(nGraphs, off.data(), fixed.data(), R.data(), t.data(), eR.data(),
			et.data(), nR.data(), nt.data(), device);
	if (rc != COSL_OK)
		throw std::runtime_error(std::string("computeNewCameraPosesBatch: ") + cosl_last_error());
	for (int c = 0; c < nGraphs; ++c)
		for (int k = 0; k < graphs[c].nNodes; ++k) {
			const size_t i = (size_t) off[c] + k;
			std::memcpy(graphs[c].poseNodes[k].newR, &nR[9 * i], sizeof(double) * 9);
			std::memcpy(graphs[c].poseNodes[k].newt, &nt[3 * i], sizeof(double) * 3);
		}
}

#endif /* SL_GLOBALPOSEESTIMATION_H_ */
