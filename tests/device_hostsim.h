// device_hostsim.h -- DeviceSim's arrays on the host (tables from csrc/device_layout.cuh) + the kernel bodies compiled
// for the emulated warp (tests/device_emu.h).  TEST INFRASTRUCTURE ONLY: shared by tests/device_step_probe.cpp (emulated engine vs
// the restatement) and tests/device_sim_emu.cpp (the real host engine / C-ABI on top of the emulated device).
#pragma once
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <vector>

#include "device_emu.h"
static struct { unsigned x = 0, y = 0, z = 0; } blockIdx;
static struct { unsigned x = 1, y = 1, z = 1; } gridDim;
using std::max;
using std::min;
namespace cfb { namespace cg = cooperative_groups; }

#include "device_sim.h"
#include "device_view.cuh"
#include "device_phases_a.cuh"
#include "device_control.cuh"   // (+ device_lc.cuh, kernels included: blockIdx / gridDim are globals here)
#include "device_phases_b.cuh"
#include "device_shard.cuh"      // the seam protocol's kernel bodies (peer-memory form), run on the emulated warp too
#include "device_layout.cuh"


namespace cfbtest {

using namespace cfb;

template <class T> struct Buf : std::vector<T> { T *p() { return this->data(); } };

struct HostSim {   // DeviceSim's arrays on the host: the static tables of device_layout.cuh, the dynamic state allocated here
    View V{};
    DeviceLayout L;
    PlanTables plans;
    LanePlanTables lanePlans;
    int P = 0, slotCap = 0;
    Buf<double> gap, remain, cust, slotCust;
    Buf<int> leader, count, pos, waitHead, waitTail, waitNext, curPhase, entCnt, ent, act0, act1, extra, blk, delStep, segIdx, cand,
        involved, spare, prio, scratch;
    Buf<unsigned char> inserted, rlAvail;
    Buf<DTmpl> tmpl;
    Buf<double2> kin, nkin, mkin;
    Buf<int4> ids, nav, slotInfo, mids, mnav;
    Buf<int2> nbuf, finSlots, veh0, veh1, shadowLog;
    Buf<Notify> notify;
    Buf<Tail> tail;
    Buf<unsigned> foeMask;
    Buf<LcSlot> lcSlot;
    Buf<SpawnRec> spawn;
    Ctrl ctrl{};
    LcCtrl lcCtrl{};
    long long steps = 0;

    void init(const RoadNet &net, double interval, bool rl, bool laneChange, double spacing) {
        L = deviceLayout(net, V, spacing);
        const int nL = V.nLanes, nK = V.nLinks, nD = V.nDrv;
        V.dt = interval; V.rl = rl ? 1 : 0;
        P = L.P;
        slotCap = 1 << 17;
        kin.resize(P); nkin.resize(P); gap.resize(P); leader.resize(P); ids.resize(P); nav.resize(P); nbuf.resize(P); cust.resize(P);
        count.resize(nD); entCnt.resize(nD); ent.resize((size_t) nD * ENT_CAP);
        waitHead.resize(std::max(nL, 1)); waitTail.resize(std::max(nL, 1)); inserted.resize(std::max(nL, 1));
        notify.resize(std::max(2 * net.nCross(), 1));
        curPhase.resize(net.nInter()); remain.resize(net.nInter()); rlAvail.resize(std::max(net.nRoadLinks(), 1));
        mkin.resize(V.moverCap); mids.resize(V.moverCap); mnav.resize(V.moverCap);
        tail.resize(nD); foeMask.resize((size_t) std::max(nK, 1) * V.maskWords);
        veh0.resize(P); veh1.resize(P); act0.resize(nD); act1.resize(nD); extra.resize(nD);
        finSlots.resize(V.finCap);
        pos.resize(slotCap); waitNext.resize(slotCap); slotInfo.resize(slotCap); slotCust.resize(slotCap); blk.resize(slotCap); delStep.resize(slotCap);
        tmpl.resize(slotCap);
        spawn.resize(1 << 14);
        segIdx.resize(P); cand.resize(LC_MAX_CAND); involved.resize(LC_MAX_CAND); shadowLog.resize(LC_MAX_CAND); prio.resize(LC_MAX_CAND);
        lcSlot.resize(slotCap); spare.resize(256); scratch.resize((size_t) 4 * LC_MAX_CAND);
        // pointers
        V.drvLength = L.drvLength.data(); V.drvMaxSpeed = L.drvMaxSpeed.data(); V.off = L.off.data();
        V.laneOutBeg = L.laneOutBeg.data(); V.laneOutLinks = L.laneOutLinks.data();
        V.llStartLane = L.llStartLane.data(); V.llEndLane = L.llEndLane.data(); V.llRoadLink = L.llRoadLink.data(); V.linkInfo = L.linkInfo.data();
        V.llCrossBeg = L.llCrossBeg.data(); V.lcIdx = L.lcIdx.data(); V.lcDist = L.lcDist.data(); V.lcPeer = L.lcPeer.data(); V.csLink = L.csLink.data();
        V.interPhaseBeg = L.interPhaseBeg.data(); V.interRLBeg = L.interRLBeg.data(); V.phaseAvailBeg = L.phaseAvailBeg.data();
        V.rlInter = L.rlInter.data(); V.phaseTime = L.phaseTime.data(); V.phaseAvail = L.phaseAvail.data(); V.interVirtual = L.interVirtual.data();
        V.tmpl = tmpl.p();
        V.kin = kin.p(); V.nkin = nkin.p(); V.gap = gap.p(); V.leader = leader.p(); V.ids = ids.p(); V.nav = nav.p(); V.nbuf = nbuf.p();
        V.count = count.p(); V.pos = pos.p(); V.waitHead = waitHead.p(); V.waitTail = waitTail.p(); V.waitNext = waitNext.p();
        V.slotInfo = slotInfo.p(); V.inserted = inserted.p(); V.notify = notify.p(); V.tail = tail.p(); V.foeMask = foeMask.p();
        V.curPhase = curPhase.p(); V.remain = remain.p(); V.rlAvail = rlAvail.p(); V.entCnt = entCnt.p(); V.ent = ent.p();
        V.mkin = mkin.p(); V.mids = mids.p(); V.mnav = mnav.p(); V.finSlots = finSlots.p();
        V.vehList[0] = veh0.p(); V.vehList[1] = veh1.p(); V.actList[0] = act0.p(); V.actList[1] = act1.p(); V.extraList = extra.p();
        V.cust = cust.p(); V.slotCust = slotCust.p(); V.blk = blk.p(); V.delStep = delStep.p(); V.ctrl = &ctrl;
        V.lcOn = laneChange ? 1 : 0;
        LcView &C = V.lc;
        C.slot = lcSlot.p(); C.segIdx = segIdx.p(); C.posDrv = L.posDrv.data(); C.segBeg = L.segBeg.data(); C.segStart = L.segStart.data();
        C.laneRoad = L.laneRoad.data(); C.laneIdx = L.laneIdx.data(); C.laneRoadN = L.laneRoadN.data(); C.laneWidth = L.laneWidth.data();
        C.cand = cand.p(); C.involved = involved.p(); C.spare = spare.p(); C.nSpare = 0; C.shadowLog = shadowLog.p(); C.ctrl = &lcCtrl;
        C.scratchA = scratch.p(); C.scratchB = scratch.p() + LC_MAX_CAND; C.scratchC = scratch.p() + 2 * LC_MAX_CAND; C.scratchD = scratch.p() + 3 * LC_MAX_CAND;
        reset();
    }
    void reset() {   // DeviceSim::reset with memset for cudaMemset
        for (const Fill &f : resetFills(V, (size_t) P, (size_t) slotCap)) memset(f.p, f.byte, f.bytes);
        std::copy(L.remain0.begin(), L.remain0.end(), remain.begin());
    }
    void setPlans(const Routing &R) {
        plans = planTables(R);
        lanePlans = lanePlanTables(R);
        V.planBeg = plans.planBeg.data(); V.planData = plans.planData.data();
        LcView &C = V.lc;
        C.planRoute = lanePlans.planRoute.data(); C.planRoadPos = lanePlans.planRoadPos.data(); C.lanePlanRoad = lanePlans.lanePlanRoad.data();
        C.lanePlanBeg = lanePlans.lanePlanBeg.data(); C.lanePlanId = lanePlans.lanePlanId.data(); C.routeLastRoad = lanePlans.routeLastRoad.data();
    }
    template <class F> void run(int nBlocks, F f) {
        gridDim.x = (unsigned) nBlocks;
        emu::launch(nBlocks, [&](int b, int n) { blockIdx.x = (unsigned) b; f(b, n); });
    }
};

}  // namespace cfbtest
