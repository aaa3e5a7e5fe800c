// device_layout.cuh -- what a DeviceSim implementation builds on the host before anything runs: the static tables of the
// lane-bucket layout, the plan tables, the device form of a vehicle template, the reset state, the debug records, and the
// index lists of a sharded run.  One definition for device_sim.cu and the emulated device of the tests (which run the
// kernel bodies over these very tables); each implementation keeps only how it allocates, fills and copies them.
//
// Host code only.  Included after device_view.cuh, like device_image.cuh.
#pragma once
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <vector>

#include "partition.h"

namespace cfb {

// Every table DeviceSim uploads once.  Tables that may be empty hold one entry of padding so that every device
// allocation is non-empty.
struct DeviceLayout {
    int P = 0;                       // positions: sum of the bucket capacities
    double spacing = 2.5;            // the vehicle spacing (length + minGap) the buckets are sized for (bucketSpacing)
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

// The spacing the lane buckets are sized for: the smallest length + minGap of the given vehicle templates, but at most
// 2.5 m (so a fleet of vehicles of 2.5 m and more, such as the grid generator's, gets the same layout whatever its
// sizes) and at least 0.5 m (a degenerate template must not size the buckets without bound).  Queued vehicles keep
// about length + minGap apart (admission: tail.dis > tail.len + minGap; car following stops minGap behind the
// leader), so a bucket of length / spacing + 8 holds a lane filled end to end.  That is a target, not an invariant
// (Lane::canEnter also admits behind a tail moving at 2 m/s or more): ERR_BUCKET_OVERFLOW stays the backstop.
inline double bucketSpacing(const std::vector<VehicleTemplate> &templates) {
    double s = 2.5;
    for (const VehicleTemplate &t : templates) s = std::min(s, t.len + t.minGap);
    return std::max(s, 0.5);
}

// Also sets V's sizes: the element counts, maskWords and the capacities moverCap, finCap and vehCap.  `spacing`:
// bucketSpacing() of the templates known when the layout is made.
inline DeviceLayout deviceLayout(const RoadNet &net, View &V, double spacing) {
    DeviceLayout L;
    L.spacing = spacing;
    const int nL = net.nLanes(), nK = net.nLinks(), nD = nL + nK, nC = net.nCross();
    V.nLanes = nL; V.nLinks = nK; V.nDrv = nD; V.nInter = net.nInter(); V.nRL = net.nRoadLinks(); V.nCross = nC;
    auto nz = [](std::vector<int> v) { if (v.empty()) v.push_back(0); return v; };
    L.drvLength.resize(nD);
    L.drvMaxSpeed.resize(nD);
    L.off.assign(nD + 1, 0);
    for (int d = 0; d < nD; ++d) {
        L.drvLength[d] = d < nL ? net.laneLength[d] : net.llLength[d - nL];
        L.drvMaxSpeed[d] = d < nL ? net.laneMaxSpeed[d] : 10000.0;  // LaneLink::maxSpeed, roadnet.h:456
        // bucket capacity: room for bumper-to-bumper traffic of vehicles `spacing` apart plus slack
        int cap = (int) (L.drvLength[d] / spacing) + 8;
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

// The static tables of the intersection observations (device_tlobs.cuh), from the layout's laneLink and phase tables
// (laneLinks are numbered intersection by intersection, roadLink by roadLink, so a roadLink's laneLinks are contiguous).
// The kernel's tables are packed into one int array; the rest are public columns of DeviceIntersectionObs.
struct IntObsLayout {
    std::vector<int> ints;   // tl | inBeg | inLane | outBeg | outLane | rlInBeg | rlInLane | rlOutBeg | rlOutLane | rlLinkBeg
    size_t tl = 0, inBeg = 0, inLane = 0, outBeg = 0, outLane = 0, rlInBeg = 0, rlInLane = 0, rlOutBeg = 0, rlOutLane = 0,
           rlLinkBeg = 0;
    int nTl = 0;
    int maxPhases = 1, maxMovements = 1;       // (at least 1: every column is non-empty)
    std::vector<int> movementBegin;            // nInter + 1: the roadLinks of intersection i (= RoadNet::interRoadLinkBeg)
    std::vector<int> movementIntersection;     // nRL
    std::vector<int> phaseCount;               // nInter, 0 for a virtual intersection
    std::vector<unsigned char> phaseMovements; // [nInter][maxPhases][maxMovements]: roadLink k of i available in phase p
    template <class Tab> void point(Tab &T, const int *at) const {
        T.nTl = nTl; T.maxPhases = maxPhases; T.tl = at + tl;
        T.inBeg = at + inBeg; T.inLane = at + inLane; T.outBeg = at + outBeg; T.outLane = at + outLane;
        T.rlInBeg = at + rlInBeg; T.rlInLane = at + rlInLane; T.rlOutBeg = at + rlOutBeg; T.rlOutLane = at + rlOutLane;
        T.rlLinkBeg = at + rlLinkBeg;
    }
    // The output ints: phase | pressure | queue | movement in | in waiting | out | inside | pressure | phase pressure |
    // lane scratch | movement begin | movement intersection | phase count.  As they stand before the first refresh:
    // phase -1 (what a virtual intersection keeps), phase pressure INT_MIN (what padding keeps), the static columns.
    size_t outInts(const View &V) const {
        return (size_t) 3 * V.nInter + 5 * (size_t) V.nRL + (size_t) V.nInter * maxPhases + V.nLanes + V.nInter + 1 +
               V.nRL + V.nInter;
    }
    std::vector<int> initialInts(const View &V) const {
        std::vector<int> v(outInts(V), 0);
        const size_t nI = V.nInter, nRL = V.nRL, pp = 3 * nI + 5 * nRL, st = pp + nI * maxPhases + V.nLanes;
        std::fill(v.begin(), v.begin() + nI, -1);
        std::fill(v.begin() + pp, v.begin() + pp + nI * maxPhases, INT_MIN);
        std::copy(movementBegin.begin(), movementBegin.end(), v.begin() + st);
        std::copy(movementIntersection.begin(), movementIntersection.end(), v.begin() + st + nI + 1);
        std::copy(phaseCount.begin(), phaseCount.end(), v.begin() + st + nI + 1 + nRL);
        return v;
    }
    // T's output columns and o's pointers, with initialInts() at `ints`, nInter doubles at `dbl` and phaseMovements at `mv`
    template <class Tab> void pointOut(Tab &T, DeviceIntersectionObs &o, const View &V, int *ints, double *dbl,
                                       unsigned char *mv) const {
        const int nI = V.nInter, nRL = V.nRL;
        T.phase = ints; T.pressure = ints + nI; T.queue = ints + 2 * nI;
        T.mvIn = ints + 3 * nI; T.mvInWaiting = T.mvIn + nRL; T.mvOut = T.mvInWaiting + nRL; T.mvInside = T.mvOut + nRL;
        T.mvPressure = T.mvInside + nRL;
        T.phasePressure = T.mvPressure + nRL;
        T.laneWait = T.phasePressure + (size_t) nI * maxPhases;
        T.remaining = dbl;
        o.phase = T.phase; o.phaseRemaining = T.remaining; o.pressure = T.pressure; o.queue = T.queue;
        o.movementIn = T.mvIn; o.movementInWaiting = T.mvInWaiting; o.movementOut = T.mvOut; o.movementInside = T.mvInside;
        o.movementPressure = T.mvPressure; o.phasePressure = T.phasePressure;
        o.movementBegin = T.laneWait + V.nLanes;
        o.movementIntersection = o.movementBegin + nI + 1;
        o.phaseCount = o.movementIntersection + nRL;
        o.phaseMovements = mv;
        o.nInter = nI; o.nRL = nRL; o.maxPhases = maxPhases; o.maxMovements = maxMovements;
    }
};
inline IntObsLayout intObsLayout(const DeviceLayout &L, const View &V) {
    IntObsLayout X;
    const int nI = V.nInter, nRL = V.nRL, nK = V.nLinks;
    std::vector<int> tl, rlLinkBeg(nRL + 1, 0);
    for (int k = 0; k < nK; ++k) rlLinkBeg[L.llRoadLink[k] + 1] += 1;
    for (int r = 0; r < nRL; ++r) rlLinkBeg[r + 1] += rlLinkBeg[r];
    // distinct lanes in first-seen order, as CSR over `n` groups of laneLinks
    auto distinct = [&](int n, auto linksOf, const std::vector<int> &lane, std::vector<int> &beg, std::vector<int> &out) {
        beg.assign(n + 1, 0);
        for (int g = 0; g < n; ++g) {
            const int k0 = linksOf(g), k1 = linksOf(g + 1);
            for (int k = k0; k < k1; ++k)
                if (std::find(out.begin() + beg[g], out.end(), lane[k]) == out.end()) out.push_back(lane[k]);
            beg[g + 1] = (int) out.size();
        }
    };
    auto interLinks = [&](int i) { return rlLinkBeg[L.interRLBeg[i]]; };
    auto rlLinks = [&](int r) { return rlLinkBeg[r]; };
    std::vector<int> inBeg, inLane, outBeg, outLane, rlInBeg, rlInLane, rlOutBeg, rlOutLane;
    distinct(nI, interLinks, L.llStartLane, inBeg, inLane);
    distinct(nI, interLinks, L.llEndLane, outBeg, outLane);
    distinct(nRL, rlLinks, L.llStartLane, rlInBeg, rlInLane);
    distinct(nRL, rlLinks, L.llEndLane, rlOutBeg, rlOutLane);
    X.phaseCount.assign(nI, 0);
    for (int i = 0; i < nI; ++i) {
        if (L.interVirtual[i]) continue;
        tl.push_back(i);
        X.phaseCount[i] = L.interPhaseBeg[i + 1] - L.interPhaseBeg[i];
        X.maxPhases = std::max(X.maxPhases, X.phaseCount[i]);
        X.maxMovements = std::max(X.maxMovements, L.interRLBeg[i + 1] - L.interRLBeg[i]);
    }
    X.nTl = (int) tl.size();
    X.movementBegin = L.interRLBeg;
    X.movementIntersection.assign(L.rlInter.begin(), L.rlInter.begin() + nRL);
    X.phaseMovements.assign((size_t) std::max(nI, 1) * X.maxPhases * X.maxMovements, 0);
    for (int i = 0; i < nI; ++i)
        for (int p = 0; p < X.phaseCount[i]; ++p)
            for (int k = 0; k < L.interRLBeg[i + 1] - L.interRLBeg[i]; ++k)
                X.phaseMovements[((size_t) i * X.maxPhases + p) * X.maxMovements + k] =
                    L.phaseAvail[L.phaseAvailBeg[L.interPhaseBeg[i] + p] + k];
    auto add = [&X](const std::vector<int> &v) { const size_t at = X.ints.size(); X.ints.insert(X.ints.end(), v.begin(), v.end()); return at; };
    X.tl = add(tl);
    X.inBeg = add(inBeg); X.inLane = add(inLane); X.outBeg = add(outBeg); X.outLane = add(outLane);
    X.rlInBeg = add(rlInBeg); X.rlInLane = add(rlInLane); X.rlOutBeg = add(rlOutBeg); X.rlOutLane = add(rlOutLane);
    X.rlLinkBeg = add(rlLinkBeg);
    return X;
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
