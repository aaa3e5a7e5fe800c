// device_layout.cuh -- what a DeviceSim implementation builds on the host before anything runs: the static tables of the
// lane-bucket layout, the plan tables, the device form of a vehicle template, the reset state, the debug records, and the
// index lists of a sharded run.  One definition for device_sim.cu and the emulated device of the tests (which run the
// kernel bodies over these very tables); each implementation keeps only how it allocates, fills and copies them.
//
// Host code only.  Included after device_view.cuh, like device_image.cuh.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

#include "partition.h"

namespace cfb {

// Every table DeviceSim uploads once.  Tables that may be empty hold one entry of padding so that every device
// allocation is non-empty.
struct DeviceLayout {
    int P = 0;                       // positions: sum of the bucket capacities
    std::vector<int> off;            // per drivable: its bucket [off[d], off[d+1])
    std::vector<double> drvLength, drvMaxSpeed;
    std::vector<int> laneOutBeg, laneOutLinks, llStartLane, llEndLane, llRoadLink;
    std::vector<int4> linkInfo;      // View::linkInfo
    std::vector<int> llCrossBeg, lcIdx, lcPeer, csLink;
    std::vector<double> lcDist;
    std::vector<int> interPhaseBeg, interRLBeg, phaseAvailBeg, rlInter;
    std::vector<double> phaseTime;
    std::vector<unsigned char> phaseAvail, interVirtual;
    std::vector<double> remain0;     // per intersection: remainDuration after TrafficLight::init(0)
    // lane change (LcView)
    std::vector<int> segBeg, laneIdx, laneRoadN, laneRoad, posDrv;
    std::vector<double> segStart, laneWidth;
};

// Also sets V's sizes: the element counts, maskWords and the capacities moverCap, finCap and vehCap.
inline DeviceLayout deviceLayout(const RoadNet &net, View &V) {
    DeviceLayout L;
    const int nL = net.nLanes(), nK = net.nLinks(), nD = nL + nK, nC = net.nCross();
    V.nLanes = nL; V.nLinks = nK; V.nDrv = nD; V.nInter = net.nInter(); V.nRL = net.nRoadLinks(); V.nCross = nC;
    auto nz = [](std::vector<int> v) { if (v.empty()) v.push_back(0); return v; };
    L.drvLength.resize(nD);
    L.drvMaxSpeed.resize(nD);
    L.off.assign(nD + 1, 0);
    for (int d = 0; d < nD; ++d) {
        L.drvLength[d] = d < nL ? net.laneLength[d] : net.llLength[d - nL];
        L.drvMaxSpeed[d] = d < nL ? net.laneMaxSpeed[d] : 10000.0;  // LaneLink::maxSpeed, roadnet.h:456
        // bucket capacity: room for bumper-to-bumper traffic of 2.5 m vehicles plus slack
        int cap = (int) (L.drvLength[d] / 2.5) + 8;
        cap = (cap + 3) & ~3;
        L.off[d + 1] = L.off[d] + cap;
    }
    L.P = L.off[nD];
    V.vehCap = L.P;
    V.moverCap = std::min(L.P, 1 << 22);
    V.finCap = 1 << 20;
    L.laneOutBeg.assign(nL + 1, 0);
    for (int l = 0; l < nL; ++l) {
        for (int ll : net.laneOutLinks[l]) L.laneOutLinks.push_back(ll);
        L.laneOutBeg[l + 1] = (int) L.laneOutLinks.size();
    }
    L.laneOutLinks = nz(L.laneOutLinks);
    // the crosses of every laneLink (CSR), and where the same cross sits in the crossing link's list
    L.llCrossBeg.assign(nK + 1, 0);
    for (int k = 0; k < nK; ++k) {
        for (const CrossRef &c : net.llCrosses[k]) {
            L.lcIdx.push_back(c.cross * 2 + c.side);
            L.lcDist.push_back(net.crossDist[c.side][c.cross]);
        }
        L.llCrossBeg[k + 1] = (int) L.lcIdx.size();
    }
    L.csLink.assign(std::max(2 * nC, 1), 0);
    for (int c = 0; c < nC; ++c) {
        L.csLink[2 * c] = net.crossLink[0][c];
        L.csLink[2 * c + 1] = net.crossLink[1][c];
    }
    std::vector<int> flatOf(std::max(2 * nC, 1), 0);
    int maxCross = 1;
    for (int k = 0; k < nK; ++k) {
        maxCross = std::max(maxCross, L.llCrossBeg[k + 1] - L.llCrossBeg[k]);
        for (int q = L.llCrossBeg[k]; q < L.llCrossBeg[k + 1]; ++q) flatOf[L.lcIdx[q]] = q;
    }
    L.lcPeer.resize(L.lcIdx.size());
    for (size_t q = 0; q < L.lcIdx.size(); ++q) L.lcPeer[q] = flatOf[L.lcIdx[q] ^ 1];
    V.maskWords = (maxCross + 31) / 32;
    if (L.lcIdx.empty()) { L.lcIdx.push_back(0); L.lcDist.push_back(0); L.lcPeer.push_back(0); }
    L.llStartLane = nz(net.llStartLane);
    L.llEndLane = nz(net.llEndLane);
    L.llRoadLink = nz(net.llRoadLink);
    L.linkInfo.assign(std::max(nK, 1), make_int4(0, 0, 0, 0));
    for (int k = 0; k < nK; ++k)
        L.linkInfo[k] = make_int4(net.llRoadLink[k], net.llEndLane[k], L.llCrossBeg[k],
                                  (net.linkIsTurn(k) ? 1 : 0) | ((int) net.rlType[net.llRoadLink[k]] << 8));
    L.interPhaseBeg = net.interPhaseBeg;
    L.interRLBeg = net.interRoadLinkBeg;
    L.phaseAvailBeg = nz(net.phaseAvailBeg);
    L.rlInter = nz(net.rlInter);
    L.phaseTime = net.phaseTime;
    if (L.phaseTime.empty()) L.phaseTime.push_back(0);
    L.phaseAvail.assign(net.phaseAvail.begin(), net.phaseAvail.end());
    if (L.phaseAvail.empty()) L.phaseAvail.push_back(0);
    L.interVirtual.assign(net.interVirtual.begin(), net.interVirtual.end());
    L.remain0.assign(net.nInter(), 0.0);
    for (int i = 0; i < net.nInter(); ++i)
        if (!net.interVirtual[i]) L.remain0[i] = net.phaseTime[net.interPhaseBeg[i]];
    // Road::buildSegmentationByInterval roadnet.cpp:687-691 with (len + minGap) * MAX_NUM_CARS_ON_SEGMENT of a
    // default VehicleInfo = (5 + 2) * 10 (roadnet.cpp:305-312, config.h:5); Lane::buildSegmentation :852-861
    L.segBeg.assign(nL + 1, 0);
    L.laneIdx.resize(nL);
    L.laneRoadN.resize(nL);
    L.laneWidth.resize(nL);
    for (int r = 0; r < net.nRoads(); ++r) {
        double len = 0.0;
        const auto &pts = net.roadPoints[r];
        for (size_t i = 0; i + 1 < pts.size(); ++i) {
            const double dx = pts[i + 1].x - pts[i].x, dy = pts[i + 1].y - pts[i].y;
            len += sqrt(dx * dx + dy * dy);
        }
        const size_t numSegs = std::max((size_t) ceil(len / ((5.0 + 2.0) * 10)), (size_t) 1);
        for (int l = net.roadLaneBeg[r]; l < net.roadLaneBeg[r + 1]; ++l) {
            L.segBeg[l] = (int) L.segStart.size();
            for (size_t i = 0; i < numSegs; ++i) L.segStart.push_back(i * net.laneLength[l] / numSegs);
            L.laneIdx[l] = net.laneIdx[l];
            L.laneRoadN[l] = net.roadNumLanes(r);
            L.laneWidth[l] = net.laneWidth[l];
        }
    }
    L.segBeg[nL] = (int) L.segStart.size();
    L.laneRoad = net.laneRoad;
    L.posDrv.resize(L.P);
    for (int d = 0; d < nD; ++d)
        for (int p = L.off[d]; p < L.off[d + 1]; ++p) L.posDrv[p] = d;
    return L;
}

// View::planBeg / planData; grown whenever a route is interned.
struct PlanTables { std::vector<int> planBeg, planData; };
inline PlanTables planTables(const Routing &R) {
    PlanTables T{R.planBeg(), R.planData()};
    if (T.planBeg.empty()) T.planBeg.push_back(0);
    if (T.planData.empty()) T.planData.push_back(PLAN_END);
    return T;
}

// LcView's plan tables (Routing::lanePlan) and routeLastRoad.
struct LanePlanTables { std::vector<int> planRoute, planRoadPos, lanePlanRoad, lanePlanBeg, lanePlanId, routeLastRoad; };
inline LanePlanTables lanePlanTables(const Routing &R) {
    auto nz = [](std::vector<int> v) { if (v.empty()) v.push_back(0); return v; };
    LanePlanTables T{nz(R.planRouteTable()), nz(R.planRoadPosTable()), nz(R.lanePlanRoadTable()), nz(R.lanePlanBegTable()),
                     nz(R.lanePlanIdTable()), std::vector<int>(std::max(R.numRoutes(), 1), -1)};
    for (int r = 0; r < R.numRoutes(); ++r) if (R.route(r).valid) T.routeLastRoad[r] = R.route(r).roads.back();
    return T;
}

inline DTmpl toDevice(const VehicleTemplate &t, double interval) {
    DTmpl d{};
    d.len = t.len;
    d.maxPosAcc = t.maxPosAcc;
    d.maxNegAcc = t.maxNegAcc;
    d.usualPosAcc = t.usualPosAcc;
    d.usualNegAcc = t.usualNegAcc;
    d.minGap = t.minGap;
    d.maxSpeed = t.maxSpeed;
    d.headwayTime = t.headwayTime;
    d.yieldDistance = t.yieldDistance;
    d.turnSpeed = t.turnSpeed;
    // vehicle.cpp:42-44 (and the identical look-ahead bound at :190-191)
    d.approachDist = t.maxSpeed * t.maxSpeed / t.usualNegAcc / 2 + t.maxSpeed * interval * 2;
    d.speed0 = t.speed;
    return d;
}

// ---- reset state: (region, byte) pairs an implementation memsets ----
struct Fill { void *p; size_t bytes; int byte; };

// What a slot without a vehicle holds: no position, no queue successor, no custom speed (NaN), no blocker, never left
// the network (delStep 0x80808080, below every step).  Slots beyond an archive's capacity are restored to this too.
inline std::vector<Fill> slotFills(const View &V, size_t S) {
    return {{V.pos, S * sizeof(int), 0xff}, {V.waitNext, S * sizeof(int), 0xff}, {V.slotCust, S * sizeof(double), 0xff},
            {V.blk, S * sizeof(int), 0xff}, {V.delStep, S * sizeof(int), 0x80}};
}
// Epoch-stamped scratch: nothing of an older timeline may match.
inline std::vector<Fill> scratchFills(const View &V) {
    return {{V.notify, (size_t) std::max(2 * V.nCross, 1) * sizeof(Notify), 0},
            {V.foeMask, (size_t) std::max(V.nLinks, 1) * V.maskWords * sizeof(unsigned), 0}};
}
// The state before the first step, apart from View::remain (DeviceLayout::remain0).  Ctrl::epoch is kept: the seam
// messages of a sharded run are stamped with it, so it never goes back.
inline std::vector<Fill> resetFills(const View &V, size_t P, size_t S) {
    const size_t nL = (size_t) std::max(V.nLanes, 1), nD = (size_t) V.nDrv, ep = offsetof(Ctrl, epoch) + sizeof(int);
    std::vector<Fill> f = {
        {V.count, nD * sizeof(int), 0}, {V.entCnt, nD * sizeof(int), 0},
        {V.waitHead, nL * sizeof(int), 0xff}, {V.waitTail, nL * sizeof(int), 0xff}, {V.inserted, nL, 0},
        {V.cust, P * sizeof(double), 0xff},
        {V.tail, nD * sizeof(Tail), 0xff},   // pos = -1: every drivable empty
        {V.curPhase, (size_t) V.nInter * sizeof(int), 0}, {V.rlAvail, (size_t) std::max(V.nRL, 1), 0},
        {V.ctrl, offsetof(Ctrl, epoch), 0}, {(char *) V.ctrl + ep, sizeof(Ctrl) - ep, 0},
    };
    for (const Fill &x : slotFills(V, S)) f.push_back(x);
    for (const Fill &x : scratchFills(V)) f.push_back(x);
    return f;
}

// ---- debug records (cfb_debug_vehicles / cfb_debug_lc_vehicles) ----
// V's off, count, leader, kin, gap, ids, nav, delStep and ctrl (and lc.slot for the lane-change records) must point to
// host memory.  A blocker that left the network in the last step is dropped lazily on the device: it is not reported.
inline int debugBlocker(const View &V, int p) {
    const int b = V.nav[p].z;
    return b >= 0 && V.delStep[b] == V.ctrl->step - 1 ? -1 : b;
}
// owned: per drivable, 0 = another rank's (only ghost data here); null = every drivable
inline void debugRecords(const View &V, const unsigned char *owned, std::vector<DebugRec> &out) {
    out.clear();
    for (int d = 0; d < V.nDrv; ++d) {
        if (owned && !owned[d]) continue;
        for (int k = 0; k < V.count[d]; ++k) {
            const int p = V.off[d] + k, lp = V.leader[p];
            DebugRec r{};
            r.slot = V.ids[p].x;
            r.drivable = d;
            r.leaderSlot = lp >= 0 ? V.ids[lp].x : -1;
            r.blockerSlot = debugBlocker(V, p);
            r.priority = V.ids[p].z;
            r.enterLaneLinkTime = V.nav[p].w;
            r.listIndex = k;
            r.dis = V.kin[p].x;
            r.speed = V.kin[p].y;
            r.gap = lp >= 0 ? V.gap[p] : 0.0;
            out.push_back(r);
        }
    }
}
inline void lcDebugRecords(const View &V, std::vector<DeviceSim::LcDebugRec> &out) {
    out.clear();
    for (int d = 0; d < V.nDrv; ++d)
        for (int k = 0; k < V.count[d]; ++k) {
            const int p = V.off[d] + k, lp = V.leader[p];
            const LcSlot &L = V.lc.slot[V.ids[p].x];
            DeviceSim::LcDebugRec r{};
            r.slot = V.ids[p].x; r.priority = V.ids[p].z; r.partnerType = L.type; r.partnerSlot = L.partner; r.drivable = d;
            r.leaderSlot = lp >= 0 ? V.ids[lp].x : -1;
            r.blockerSlot = debugBlocker(V, p);
            r.flags = L.changing | (L.finished << 1);
            r.lastDir = L.lastDir;
            r.dis = V.kin[p].x; r.speed = V.kin[p].y; r.gap = lp >= 0 ? L.gap : 0.0;
            r.offset = L.offset; r.waiting = L.waiting; r.lastChange = L.lastChange;
            out.push_back(r);
        }
}

// ---- sharded mode (partition.h) ----
// What configureShard hands to the kernels: k_ingest's index lists and the boundary lanes of every peer.
struct ShardLists {
    std::vector<unsigned char> owned;   // View::owned: 1 = owned, 2 = a lane this rank feeds (ghost copy), 0 = foreign
    std::vector<int> ing;               // lanes owned or fed | laneLinks owned | roadLinks owned, one entry of padding
    std::vector<int> boundOut, boundIn; // all peers concatenated, padded to one entry
    std::vector<int> outBeg, inBeg;     // per peer: where its lanes start in boundOut / boundIn
    int nIngLanes = 0, nIngLinks = 0, nIngRL = 0, nBoundOut = 0, nBoundIn = 0;
    // the View fields, with ing / boundOut / boundIn where the implementation keeps the three lists
    void point(View &V, const int *ingAt, const int *boundOutAt, const int *boundInAt) const {
        V.nIngLanes = nIngLanes; V.nIngLinks = nIngLinks; V.nIngRL = nIngRL;
        V.ingLanes = ingAt; V.ingLinks = ingAt + nIngLanes; V.ingRL = ingAt + nIngLanes + nIngLinks;
        V.nBoundOut = nBoundOut; V.nBoundIn = nBoundIn;
        V.boundOut = boundOutAt; V.boundIn = boundInAt;
    }
};
inline ShardLists shardLists(int nLanes, int nLinks, const std::vector<unsigned char> &owned,
                             const std::vector<std::vector<int>> &feedPerPeer, const std::vector<std::vector<int>> &ownPerPeer,
                             const std::vector<unsigned char> &ownedRoadLinks) {
    ShardLists S;
    const int world = (int) feedPerPeer.size();
    S.owned = owned;
    for (int q = 0; q < world; ++q)
        for (int l : feedPerPeer[q]) S.owned[l] = 2;   // ghost lanes: admitted into locally, never listed as work
    // k_ingest walks these instead of every lane / laneLink / roadLink of the whole network
    for (int l = 0; l < nLanes; ++l) if (S.owned[l]) S.ing.push_back(l);
    S.nIngLanes = (int) S.ing.size();
    for (int k = 0; k < nLinks; ++k) if (owned[nLanes + k]) S.ing.push_back(k);
    S.nIngLinks = (int) S.ing.size() - S.nIngLanes;
    for (int r = 0; r < (int) ownedRoadLinks.size(); ++r) if (ownedRoadLinks[r]) S.ing.push_back(r);
    S.nIngRL = (int) S.ing.size() - S.nIngLanes - S.nIngLinks;
    S.ing.push_back(0);
    S.outBeg.assign(1, 0);
    S.inBeg.assign(1, 0);
    for (int q = 0; q < world; ++q) {
        S.boundOut.insert(S.boundOut.end(), feedPerPeer[q].begin(), feedPerPeer[q].end());
        S.boundIn.insert(S.boundIn.end(), ownPerPeer[q].begin(), ownPerPeer[q].end());
        S.outBeg.push_back((int) S.boundOut.size());
        S.inBeg.push_back((int) S.boundIn.size());
    }
    S.nBoundOut = (int) S.boundOut.size();
    S.nBoundIn = (int) S.boundIn.size();
    if (S.boundOut.empty()) S.boundOut.push_back(0);
    if (S.boundIn.empty()) S.boundIn.push_back(0);
    return S;
}

// The seam index tables of the peer-memory transport (seamTables, partition.h) packed into one int array:
// nbr | outPeer | outDst | inPeer | inDst | ticket[2].
struct SeamIndex {
    std::vector<int> ints;
    int nNbr = 0;
    size_t outPeer = 0, outDst = 0, inPeer = 0, inDst = 0, ticket = 0;
    // ShardP2P's index pointers (device_shard.cuh), with `ints` at `at`
    template <class P2P> void point(P2P &S, int *at) const {
        S.nbr = at; S.nNbr = nNbr;
        S.outPeer = at + outPeer; S.outDst = at + outDst; S.inPeer = at + inPeer; S.inDst = at + inDst;
        S.ticket = at + ticket;
    }
};
inline SeamIndex seamIndex(const SeamTables &T) {
    SeamIndex X;
    auto add = [&X](const std::vector<int> &v) { const size_t at = X.ints.size(); X.ints.insert(X.ints.end(), v.begin(), v.end()); return at; };
    X.nNbr = (int) T.nbr.size();
    add(T.nbr);
    X.outPeer = add(T.outPeer);
    X.outDst = add(T.outDst);
    X.inPeer = add(T.inPeer);
    X.inDst = add(T.inDst);
    X.ticket = add({0, 0});
    return X;
}

}  // namespace cfb
