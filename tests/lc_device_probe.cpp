// CPU probe: the device code of the control phase and of the lane-change DRAFT, compiled for the HOST.
//
// csrc/device_control.cuh (canPass, phase_control = the body of k_control) and csrc/device_lc.cuh
// (lcInitSegments, lcMakeSignal, lcSchedule incl. shadow insertion, lcControlTail) are plain functions over
// the lane-bucket arrays of csrc/device_view.cuh.  With the CUDA keywords defined away and one-thread
// stand-ins for the few execution-model calls they use (atomics, coalesced_threads, __ffs), they run here
// on arrays built from the restatement's state, hooked into its step (oracle/cityflow_oracle.cpp, device
// form), and must decide exactly what the restatement decides, every step:
//   * before / after its lane-change phases: who signals where, who receives whose signal, target leader /
//     follower and gaps, who starts changing, list position and route plan of every new shadow;
//   * before / after its control pass: next speed and next distance (bit for bit), next drivable, blocker
//     and mover staging of EVERY vehicle -- through phase_control itself, with this step's Cross::notify
//     results taken from the restatement -- plus, with lane change, offset progress, finish / abort and
//     partner links of the involved vehicles (the sequential tail).
// The restatement is pinned against the compiled reference (and against oracle/_ref/refdump_lcorder for lane
// change).  What this does NOT cover: k_notify / k_move / k_leader, launch plumbing, host bookkeeping.
//
//   g++ -std=c++17 -O1 -ffp-contract=off -I/usr/local/cuda/include -Icityflow_b200/csrc tests/lc_device_probe.cpp \
//       cityflow_b200/csrc/roadnet.cpp cityflow_b200/csrc/flows.cpp -o probe && ./probe config.json steps
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <vector>

#include "device_emu.h"   // CUDA keywords defined away + stand-ins; this probe runs everything as ONE thread, no fibers
#define CFB_LC_HOST_PROBE 1
using std::max;
using std::min;
namespace cfb { namespace cg = cooperative_groups; }

#include "device_sim.h"
#include "device_view.cuh"
#include "device_phases_a.cuh"   // headSearch (the warp code in there is not run by this probe)
#include "device_control.cuh"   // canPass, phase_control (+ device_lc.cuh)
#include "device_layout.cuh"    // the product's static tables; the buckets (off, posDrv) are this probe's own

#include "../oracle/cityflow_oracle.cpp"   // Oracle / Veh (anonymous namespace: visible in this translation unit)

namespace {

using namespace cfb;

struct Soa {   // the arrays the device functions touch, sized for this step
    std::vector<int> off, count, pos, leader, segIdx, posDrv, cand, involved, spare, act[2], blk, extra, entCnt, ent, delStep;
    std::vector<double> gap, cust;
    PlanTables plans;
    LanePlanTables lanePlans;
    std::vector<unsigned> foeMask;
    std::vector<Notify> notify;
    std::vector<unsigned char> rlAvail;
    std::vector<Veh *> allVeh;
    std::vector<double2> kin, mkin, nkin;
    std::vector<int2> nbuf;
    std::vector<Veh *> involvedVeh;
    std::vector<int4> ids, nav, mids, mnav;
    std::vector<int2> veh[2], shadowLog;
    std::vector<Tail> tail;
    std::vector<DTmpl> tmpl;
    std::vector<LcSlot> slot;
    std::vector<Veh *> vehOfSlot;
    std::map<Veh *, int> slotOf;
    Ctrl ctrl{};
    LcCtrl lcCtrl{};
    View V{};
    int epoch = 0;
};

Soa *g = nullptr;
DeviceLayout g_layout;   // deviceLayout() of the restatement's road network ...
View g_sized;            // ... and the View sizes it sets
static int slotAt(Soa &S, Veh *v, const char *what) {
    auto it = S.slotOf.find(v);
    if (it == S.slotOf.end()) { printf("PROBE: %s refers to a vehicle that is not running (prio %d, running %d)\n", what, v->priority, (int) v->running); fflush(stdout); abort(); }
    return it->second;
}
long long g_checked = 0, g_candidates = 0, g_shadows = 0, g_steps = 0, g_involved = 0, g_controls = 0;
int g_fail = 0;

#define CHECK(cond, ...)                                  \
    do {                                                  \
        if (!(cond)) {                                    \
            if (g_fail < 10) { printf("FAIL step %zu: ", o.step + 1); printf(__VA_ARGS__); printf("\n"); } \
            ++g_fail;                                     \
        }                                                 \
    } while (0)

void build(Oracle &o, bool forControl) {
    delete g;
    g = new Soa();
    Soa &S = *g;
    const RoadNet &net = o.net;
    const DeviceLayout &L = g_layout;
    const int nL = net.nLanes(), nD = net.nDrivables();
    S.epoch = (int) o.step + 1;
    // buckets: list size + headroom
    S.off.assign(nD + 1, 0);
    for (int d = 0; d < nD; ++d) S.off[d + 1] = S.off[d] + (int) o.lists[d].size() + 6;
    const int P = S.off[nD];
    S.count.assign(nD, 0);
    S.kin.assign(P, make_double2(0, 0)); S.ids.assign(P, make_int4(0, 0, 0, 0)); S.nav.assign(P, make_int4(0, 0, 0, 0));
    S.gap.assign(P, 0); S.cust.assign(P, 0); S.segIdx.assign(P, 0); S.leader.assign(P, -1); S.posDrv.assign(P, 0);
    for (int d = 0; d < nD; ++d) for (int p = S.off[d]; p < S.off[d + 1]; ++p) S.posDrv[p] = d;
    // slots and per-vehicle records
    int nSlots = 0;
    for (auto &kv : o.pool) if (kv.second->running) { S.slotOf[kv.second] = nSlots++; S.vehOfSlot.push_back(kv.second); }
    const int nSpare = 64;
    S.slot.assign(nSlots + nSpare, LcSlot{});
    S.pos.assign(nSlots + nSpare, -1);
    S.blk.assign(nSlots + nSpare, -1);
    S.tmpl.resize(nSlots + nSpare);
    for (int k = 0; k < nSpare; ++k) S.spare.push_back(nSlots + k);
    // plans: every vehicle gets "the plan from its current lane" of its route (Routing::lanePlan)
    Routing &R = *o.routing;
    for (int d = 0; d < nD; ++d) {
        int k = 0;
        for (Veh *v : o.lists[d]) {
            const int p = S.off[d] + k++;
            const int s = S.slotOf.at(v);
            int plan = 0, planIdx = 0, next = -1;
            if (!o.isLink(d)) {
                const int route = R.intern(v->route);
                plan = R.lanePlan(route, v->iCur, net.laneIdx[d]);
                planIdx = R.planBeg()[plan];
                next = R.planData()[planIdx + 1];
                const int want = o.nextDrivable(*v);
                if (!(next == want || (next < 0 && want < 0))) { printf("PROBE: plan disagrees with the router (%d vs %d)\n", next, want); ++g_fail; }
            } else {   // on a laneLink: second entry of the plan from the lane it came from
                const int route = R.intern(v->route);
                plan = R.lanePlan(route, v->iCur, net.laneIdx[v->prevDrivable]);
                planIdx = R.planBeg()[plan] + 1;
                next = R.planData()[planIdx + 1];
                if (R.planData()[planIdx] != d || next != o.nextDrivable(*v)) { printf("PROBE: link plan disagrees with the router\n"); ++g_fail; }
            }
            S.kin[p] = make_double2(v->dis, v->t.speed);
            S.ids[p] = make_int4(s, s, v->priority, next);
            S.nav[p] = make_int4(planIdx, v->prevDrivable, v->blocker ? slotAt(S, v->blocker, "blocker(nav)") : -1, (int) v->enterLaneLinkTime);
            S.gap[p] = v->gap;
            S.cust[p] = v->bCustomSet ? v->bCustom : NAN;
            S.pos[s] = p;
            S.tmpl[s] = toDevice(v->t, o.interval);
            S.allVeh.push_back(v);
            LcSlot &L = S.slot[s];
            lcResetSlot(L, plan);
            L.partner = v->partner ? slotAt(S, v->partner, "partner") : -1;
            L.type = v->partnerType; L.changing = v->changing; L.finished = v->lcFinished;
            if (v->sigSend) { L.sendTarget = v->sigSend->target; L.sendDir = v->sigSend->direction; }   // only changing vehicles still hold one here
            L.offset = v->offset; L.waiting = v->waitingTime; L.lastChange = v->lastChangeTime; L.gap = v->gap; L.lastDir = v->lastDir;
            // (only meaningful when built after scheduling, for the control phase)
            if (v->sigSend && !v->changing) L.sendEpoch = S.epoch;
            if (v->sigRecv) { L.recvEpoch = S.epoch; }
            L.leaderGap = v->leaderGap; L.followerGap = v->followerGap;
            L.head = v->ctlHead;
        }
        S.count[d] = k;
    }
    S.plans = planTables(R);
    S.lanePlans = lanePlanTables(R);
    S.tail.resize(nD);
    for (int d = 0; d < nD; ++d) {
        Tail t{}; t.pos = -1; t.prev = -1;
        if (S.count[d] > 0) {
            const int q = S.off[d] + S.count[d] - 1;
            t.dis = S.kin[q].x; t.speed = S.kin[q].y; t.len = S.tmpl[S.ids[q].y].len; t.pos = q; t.prev = S.nav[q].y;
        }
        S.tail[d] = t;
    }
    for (int par = 0; par < 2; ++par) { S.veh[par].assign(P + 64, make_int2(0, 0)); S.act[par].assign(nD + 8, 0); }
    S.cand.assign(LC_MAX_CAND, 0); S.involved.assign(LC_MAX_CAND, 0); S.shadowLog.assign(LC_MAX_CAND, make_int2(0, 0));
    S.nkin.assign(P, make_double2(0, 0)); S.nbuf.assign(P, make_int2(-1, -1));
    S.mkin.assign(8192, make_double2(0, 0)); S.mids.assign(8192, make_int4(0, 0, 0, 0)); S.mnav.assign(8192, make_int4(0, 0, 0, 0));
    S.entCnt.assign(nD, 0); S.ent.assign((size_t) nD * ENT_CAP, 0); S.extra.assign(nD + 8, 0);
    View &V = S.V;
    V = g_sized;
    V.dt = o.interval; V.par = 0; V.vehCap = P + 64;
    V.drvLength = L.drvLength.data(); V.off = S.off.data(); V.laneOutBeg = L.laneOutBeg.data(); V.laneOutLinks = L.laneOutLinks.data();
    V.llStartLane = L.llStartLane.data();   // headSearch (the shadow's immediate leader update)
    V.tmpl = S.tmpl.data(); V.planBeg = S.plans.planBeg.data(); V.planData = S.plans.planData.data();
    V.kin = S.kin.data(); V.gap = S.gap.data(); V.leader = S.leader.data(); V.ids = S.ids.data(); V.nav = S.nav.data();
    V.count = S.count.data(); V.pos = S.pos.data(); V.tail = S.tail.data(); V.cust = S.cust.data(); V.blk = S.blk.data();
    V.vehList[0] = S.veh[0].data(); V.vehList[1] = S.veh[1].data(); V.actList[0] = S.act[0].data(); V.actList[1] = S.act[1].data();
    S.ctrl.step = (int) o.step;
    V.ctrl = &S.ctrl;
    V.nkin = S.nkin.data(); V.nbuf = S.nbuf.data(); V.mkin = S.mkin.data(); V.mids = S.mids.data(); V.mnav = S.mnav.data();
    V.entCnt = S.entCnt.data(); V.ent = S.ent.data(); V.extraList = S.extra.data(); V.moverCap = 8192;
    V.lcOn = 1;
    LcView &C = V.lc;
    C.slot = S.slot.data(); C.segIdx = S.segIdx.data(); C.posDrv = S.posDrv.data(); C.segBeg = L.segBeg.data(); C.segStart = L.segStart.data();
    C.laneIdx = L.laneIdx.data(); C.laneRoadN = L.laneRoadN.data(); C.laneWidth = L.laneWidth.data();
    C.planRoute = S.lanePlans.planRoute.data(); C.planRoadPos = S.lanePlans.planRoadPos.data();
    C.lanePlanRoad = S.lanePlans.lanePlanRoad.data(); C.lanePlanBeg = S.lanePlans.lanePlanBeg.data(); C.lanePlanId = S.lanePlans.lanePlanId.data();
    C.routeLastRoad = S.lanePlans.routeLastRoad.data(); C.laneRoad = L.laneRoad.data();
    C.cand = S.cand.data(); C.involved = S.involved.data(); C.spare = S.spare.data(); C.nSpare = nSpare;
    C.shadowLog = S.shadowLog.data(); C.ctrl = &S.lcCtrl;

    // ---- what the control phase needs on top ----
    const int nK = net.nLinks();
    std::vector<int> flatOf(std::max(2 * net.nCross(), 1), 0);   // where each cross side sits in the cross lists
    for (int q = 0; q < L.llCrossBeg[nK]; ++q) flatOf[L.lcIdx[q]] = q;
    // this step's notifications (Cross::notify, engine.cpp:317-372) straight from the restatement
    // (before notifyCross has run they are last step's and may point to vehicles that are gone)
    S.notify.assign(std::max(2 * net.nCross(), 1), Notify{0.0, -1, -1});
    S.foeMask.assign((size_t) std::max(nK, 1) * V.maskWords, 0u);
    for (int c = 0; forControl && c < net.nCross(); ++c)
        for (int side = 0; side < 2; ++side) {
            Veh *nv = o.notifyVeh[side][c];
            if (!nv) continue;
            const int cs = 2 * c + side;
            S.notify[cs] = Notify{o.notifyDist[side][c], S.pos[slotAt(S, nv, "notify")], S.epoch};
            const int foeLink = L.csLink[cs ^ 1];
            const int bit = flatOf[cs ^ 1] - L.llCrossBeg[foeLink];
            S.foeMask[(size_t) foeLink * V.maskWords + (bit >> 5)] |= 1u << (bit & 31);
        }
    S.rlAvail.assign(std::max(net.nRoadLinks(), 1), 0);
    for (int k = 0; k < nK; ++k) S.rlAvail[net.llRoadLink[k]] = o.linkAvailable(k) ? 1 : 0;
    S.delStep.assign(S.pos.size(), INT_MIN);
    int nVeh = 0, nCustom = 0;
    for (int d = 0; d < nD; ++d) {
        int k = 0;
        for (Veh *v : o.lists[d]) {
            const int p = S.off[d] + k++;
            S.leader[p] = v->leader ? S.pos[slotAt(S, v->leader, "leader")] : -1;
            S.blk[S.slotOf.at(v)] = v->blocker ? slotAt(S, v->blocker, "blocker") : -1;
            S.veh[0][nVeh++] = make_int2(p, d);
            nCustom += v->bCustomSet;
        }
    }
    S.ctrl.nVeh[0] = nVeh;
    S.ctrl.nCustom = nCustom;
    V.drvMaxSpeed = L.drvMaxSpeed.data(); V.linkInfo = L.linkInfo.data(); V.llCrossBeg = L.llCrossBeg.data(); V.lcIdx = L.lcIdx.data();
    V.lcDist = L.lcDist.data(); V.csLink = L.csLink.data(); V.foeMask = S.foeMask.data(); V.notify = S.notify.data();
    V.rlAvail = S.rlAvail.data(); V.delStep = S.delStep.data();
    V.lcOn = o.laneChange ? 1 : 0;
    // the foe half of Cross::canPass, as k_notify attaches it to every notification (device_control.cuh foeTerms)
    for (int cs = 0; forControl && cs < 2 * net.nCross(); ++cs)
        if (S.notify[cs].epoch == S.epoch && S.notify[cs].pos >= 0) foeTerms(V, S.notify[cs], L.linkInfo[L.csLink[cs]].w);
}

void before(Oracle &o) {
    build(o, false);
    Soa &S = *g;
    View &V = S.V;
    for (int l = 0; l < V.nLanes; ++l) lcInitSegments(V, V.lc, l);
    for (int d = 0; d < V.nDrv; ++d)
        for (int k = 0; k < S.count[d]; ++k) lcMakeSignal(V, V.lc, S.off[d] + k, d, S.epoch);
    lcSchedule(V, V.lc, S.epoch);
}

void after(Oracle &o) {
    Soa &S = *g;
    View &V = S.V;
    const int epoch = S.epoch;
    ++g_steps;
    CHECK(S.lcCtrl.error == 0, "capacity error %d", S.lcCtrl.error);
    // shadows: the restatement's new shadows <-> the device's, by parent
    int newShadows = 0;
    for (auto &kv : o.pool) {
        Veh *v = kv.second;
        if (!v->running || S.slotOf.count(v)) continue;
        ++newShadows;                                      // created by this step's scheduling
        CHECK(v->partnerType == 2 && v->partner && S.slotOf.count(v->partner), "new vehicle that is not a shadow");
        const int ps = S.slotOf.at(v->partner);
        const int sh = S.slot[ps].partner;
        CHECK(sh >= 0 && S.slot[ps].type == 1 && S.slot[sh].type == 2 && S.slot[sh].partner == ps, "parent %d has no shadow on the device", v->partner->priority);
        if (sh >= 0) { S.slotOf[v] = sh; if ((int) S.vehOfSlot.size() <= sh) S.vehOfSlot.resize(sh + 1, nullptr); S.vehOfSlot[sh] = v; }
    }
    CHECK(newShadows == S.lcCtrl.nShadows, "shadows: restatement %d device %d", newShadows, S.lcCtrl.nShadows);
    g_shadows += newShadows;
    // the log must be in the restatement's creation order (= RNG order): ascending shadow creation is the
    // order of priorities drawn, which the restatement recorded implicitly in its own draws; compare by
    // walking the device's log and checking each parent got its shadow
    for (int k = 0; k < S.lcCtrl.nShadows; ++k) CHECK(S.slot[S.shadowLog[k].x].partner == S.shadowLog[k].y, "shadow log entry %d inconsistent", k);
    // lists: same vehicles in the same order on every drivable
    for (int d = 0; d < V.nDrv; ++d) {
        CHECK((int) o.lists[d].size() == S.count[d], "drivable %d: %zu vs %d vehicles", d, o.lists[d].size(), S.count[d]);
        if ((int) o.lists[d].size() != S.count[d]) continue;
        int k = 0;
        for (Veh *v : o.lists[d]) {
            const int p = S.off[d] + k++;
            const int s = S.slotOf.count(v) ? S.slotOf.at(v) : -1;
            CHECK(S.ids[p].x == s && S.pos[s] == p, "drivable %d position %d: slot %d vs %d", d, k - 1, S.ids[p].x, s);
            CHECK(S.kin[p].x == v->dis && S.kin[p].y == v->t.speed, "drivable %d position %d: kinematics differ", d, k - 1);
            if (!o.isLink(d)) CHECK(S.segIdx[p] == (int) v->segIndex, "segment index of prio %d: %d vs %zu", v->priority, S.segIdx[p], v->segIndex);
            ++g_checked;
        }
        if (S.count[d] > 0) {
            const Tail &t = S.tail[d];
            Veh *last = o.lists[d].back();
            CHECK(t.pos == S.off[d] + S.count[d] - 1 && t.dis == last->dis && t.len == last->t.len, "tail record of drivable %d", d);
        }
    }
    // per-vehicle lane-change state
    int cands = 0;
    for (auto &kv : S.slotOf) {
        Veh *v = kv.first;
        const LcSlot &L = S.slot[kv.second];
        const bool send = v->sigSend != nullptr;
        CHECK(send == lcSendValid(L, epoch), "prio %d: signalSend %d vs %d", v->priority, send, lcSendValid(L, epoch));
        if (send && lcSendValid(L, epoch)) {
            CHECK(v->sigSend->target == L.sendTarget && v->sigSend->direction == L.sendDir, "prio %d: target %d/%d dir %d/%d", v->priority,
                  v->sigSend->target, L.sendTarget, v->sigSend->direction, L.sendDir);
        }
        const bool recv = v->sigRecv != nullptr;
        CHECK(recv == lcRecvValid(L, epoch), "prio %d: signalRecv %d vs %d", v->priority, recv, lcRecvValid(L, epoch));
        if (recv && lcRecvValid(L, epoch)) CHECK(S.slotOf.at(v->sigRecv->source) == L.recvSrc, "prio %d: signal source", v->priority);
        CHECK((int) v->changing == L.changing && v->partnerType == L.type, "prio %d: changing %d/%d type %d/%d", v->priority, v->changing, L.changing, v->partnerType, L.type);
        CHECK((v->partner ? S.slotOf.at(v->partner) : -1) == L.partner, "prio %d: partner", v->priority);
        CHECK(v->waitingTime == L.waiting, "prio %d: waiting time %g vs %g", v->priority, v->waitingTime, L.waiting);
        if (v->planChange() && v->isReal()) {   // a candidate: neighbours and gaps were computed
            ++cands;
            const int tl = v->targetLeader ? S.slotOf.at(v->targetLeader) : -1, tf = v->targetFollower ? S.slotOf.at(v->targetFollower) : -1;
            CHECK(L.tgtEpoch == epoch && L.tgtLeader == tl && L.tgtFollower == tf, "prio %d: target leader %d/%d follower %d/%d", v->priority, tl, L.tgtLeader, tf, L.tgtFollower);
            CHECK(L.leaderGap == v->leaderGap && L.followerGap == v->followerGap, "prio %d: gaps %g/%g %g/%g", v->priority, v->leaderGap, L.leaderGap, v->followerGap, L.followerGap);
        }
        if (v->partnerType == 2 && !v->sigSend) {   // a shadow: plan continues the parent's route from the new lane
            const int p = S.pos[kv.second];
            const int want = o.nextDrivable(*v);
            CHECK(S.ids[p].w == want || (S.ids[p].w < 0 && want < 0), "shadow prio %d: next drivable %d vs %d", v->priority, S.ids[p].w, want);
        }
    }
    CHECK(cands == S.lcCtrl.nCand, "candidates: restatement %d device %d", cands, S.lcCtrl.nCand);
    g_candidates += cands;
}

// ---- control tail: engine.cpp:195-244 for the vehicles involved in a lane change ------------------------
void beforeControl(Oracle &o) {
    build(o, true);
    Soa &S = *g;
    View &V = S.V;
    const int epoch = S.epoch;
    // second pass over the slots: the fields that refer to other vehicles, and this step's neighbours
    for (auto &kv : S.slotOf) {
        Veh *v = kv.first;
        LcSlot &L = S.slot[kv.second];
        if (v->sigRecv) L.recvSrc = S.slotOf.at(v->sigRecv->source);
        if (v->isReal() && v->planChange()) {
            L.tgtEpoch = epoch;
            L.tgtLeader = v->targetLeader ? S.slotOf.at(v->targetLeader) : -1;
            L.tgtFollower = v->targetFollower ? S.slotOf.at(v->targetFollower) : -1;
        }
    }
    // the real control phase, one vehicle after the other: the lane-change hook leaves the involved ones to the tail
    blockDim.x = 1; threadIdx.x = 0;   // one vehicle after the other
    phase_control(V, 0, 1);
    for (int k = 0; k < S.lcCtrl.nInvolved; ++k) S.involvedVeh.push_back(S.vehOfSlot[S.involved[k]]);
    if (o.laneChange) lcControlTail(V, V.lc, epoch);
}

void afterControl(Oracle &o) {
    Soa &S = *g;
    for (Veh *v : S.allVeh) {   // every running vehicle: the buffers k_move will commit
        const int s = S.slotOf.at(v);
        const int p = S.pos[s];
        const double2 nk = S.nkin[p];
        const int2 nb = S.nbuf[p];
        CHECK(v->bSpeedSet && nk.y == v->bSpeed, "prio %d: next speed %.17g vs %.17g", v->priority, v->bSpeed, nk.y);
        CHECK(v->bDisSet && nk.x == v->bDis, "prio %d: next distance %.17g vs %.17g", v->priority, v->bDis, nk.x);
        const int want = v->bEndSet ? -2 : (v->bDrvSet && v->bDrv >= 0 ? v->bDrv : -1);
        CHECK(nb.x == want, "prio %d: next drivable %d vs %d (on drivable %d of %d lanes, dis %.3f, plan next %d, plan %d idx %d)", v->priority, want, nb.x,
              v->drivable, S.V.nLanes, v->dis, S.ids[p].w, S.slot[s].plan, S.nav[p].x);
        CHECK(nb.y == (v->bBlockerSet && v->bBlocker ? S.slotOf.at(v->bBlocker) : -1), "prio %d: blocker buffer", v->priority);
        if (o.laneChange) CHECK(v->waitingTime == S.slot[s].waiting, "prio %d: waiting time %g vs %g", v->priority, v->waitingTime, S.slot[s].waiting);
        ++g_controls;
    }
    for (Veh *v : S.involvedVeh) {
        const int s = S.slotOf.at(v);
        const LcSlot &L = S.slot[s];
        const int p = S.pos[s];
        const double2 nk = S.nkin[p];
        const int2 nb = S.nbuf[p];
        CHECK(v->bSpeedSet && nk.y == v->bSpeed, "prio %d: next speed %.17g vs %.17g", v->priority, v->bSpeed, nk.y);
        CHECK(v->bDisSet && nk.x == v->bDis, "prio %d: next distance %.17g vs %.17g", v->priority, v->bDis, nk.x);
        const int want = v->bEndSet ? -2 : (v->bDrvSet && v->bDrv >= 0 ? v->bDrv : -1);
        CHECK(nb.x == want, "prio %d: next drivable %d vs %d", v->priority, want, nb.x);
        CHECK(nb.y == (v->bBlockerSet && v->bBlocker ? S.slotOf.at(v->bBlocker) : -1), "prio %d: blocker buffer", v->priority);
        CHECK(v->offset == L.offset && (int) v->changing == L.changing && (int) v->lcFinished == L.finished, "prio %d: offset %g/%g changing %d/%d finished %d/%d",
              v->priority, v->offset, L.offset, v->changing, L.changing, v->lcFinished, L.finished);
        CHECK(v->partnerType == L.type && (v->partner ? S.slotOf.at(v->partner) : -1) == L.partner, "prio %d: partner link after control", v->priority);
        CHECK(v->waitingTime == L.waiting && v->lastChangeTime == L.lastChange, "prio %d: waiting %g/%g last change %g/%g", v->priority, v->waitingTime,
              L.waiting, v->lastChangeTime, L.lastChange);
        if (want >= 0) {   // staged for its new drivable (engine.cpp:247-249)
            bool found = false;
            for (int k = 0; k < S.entCnt[want] && k < ENT_CAP; ++k) {
                const int m = S.ent[(size_t) want * ENT_CAP + k];
                if (S.mids[m].x == s) { found = S.mkin[m].x == v->bDis && S.mkin[m].y == v->bSpeed && S.mnav[m].y == v->drivable; }
            }
            CHECK(found, "prio %d: not staged for drivable %d", v->priority, want);
        }
        ++g_involved;
    }
    CHECK(S.ctrl.error == 0, "device error flags %d", S.ctrl.error);
}

void probe(Oracle &o, int phase) {
    if (phase == 0) before(o);
    else if (phase == 1) after(o);
    else if (phase == 2) beforeControl(o);
    else afterControl(o);
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) { fprintf(stderr, "usage: lc_device_probe config.json steps\n"); return 64; }
    Oracle o;
    if (!o.load(argv[1])) { fprintf(stderr, "cannot load %s\n", argv[1]); return 2; }
    o.routing->enableLanePlans();
    g_layout = deviceLayout(o.net, g_sized);
    o.lcProbe = probe;
    o.deviceForm = true;   // (proven equal to the reference order; gives the hook between the two control passes)
    const int steps = atoi(argv[2]);
    for (int s = 0; s < steps && g_fail == 0; ++s) o.nextStep();
    printf("%s %lld steps, %lld list entries, %lld candidates, %lld shadows checked, %lld control tails, %lld controls, %d failures\n",
           g_fail ? "FAIL" : "OK", g_steps, g_checked, g_candidates, g_shadows, g_involved, g_controls, g_fail);
    return g_fail ? 1 : 0;
}
