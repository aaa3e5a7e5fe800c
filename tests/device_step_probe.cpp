// CPU probe: the WHOLE device step on the host.  TEST INFRASTRUCTURE ONLY.
//
// The bodies of all five step kernels (csrc/device_phases_a.cuh: k_ingest, k_notify; device_control.cuh:
// k_control; device_phases_b.cuh: k_move, k_leader) and, with laneChange, the lane-change kernels
// (csrc/device_lc.cuh) run on an emulated warp (tests/device_emu.h: 32 lock-stepped fibers) over
// persistent lane-bucket arrays laid out by DeviceSim's own layout code (csrc/device_layout.cuh).  The emulated
// engine gets the same spawn events as the restatement (oracle/cityflow_oracle.cpp) and evolves ON ITS OWN; after
// every step its full state --
// list order, distance, speed, leader, gap, blocker, enterLaneLinkTime of every vehicle, vehicle counts,
// finished vehicles, and with laneChange every shadow, partner link, offset, waiting time -- must equal the
// restatement's.  That is the GPU parity test (tests/test_gpu_parity.py) minus the GPU: it checks the
// kernels' logic and their interplay, not launch configuration, streams or the host engine.
//
//   g++ -std=c++17 -O1 -ffp-contract=off -I/usr/local/cuda/include -Icityflow_b200/csrc tests/device_step_probe.cpp \
//       cityflow_b200/csrc/roadnet.cpp cityflow_b200/csrc/flows.cpp -o probe && ./probe config.json steps
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <vector>

#include "device_hostsim.h"

#include "../oracle/cityflow_oracle.cpp"

namespace {

using namespace cfb;

using cfbtest::HostSim;

HostSim *S = nullptr;
std::map<Veh *, int> slotOf;
std::vector<Veh *> vehOfSlot;
int g_nextSlot = 0, g_fail = 0;
long long g_checked = 0, g_shadows = 0, g_finished = 0;

#define CHECK(cond, ...)                                                                            \
    do {                                                                                            \
        if (!(cond)) {                                                                              \
            if (g_fail < 12) { printf("FAIL step %zu: ", o.step); printf(__VA_ARGS__); printf("\n"); } \
            ++g_fail;                                                                               \
        }                                                                                           \
    } while (0)

int newSlot(Veh *v) {
    const int s = g_nextSlot++;
    if (s >= S->slotCap) { printf("probe: out of slots\n"); exit(3); }
    slotOf[v] = s;
    if ((int) vehOfSlot.size() <= s) vehOfSlot.resize(s + 1, nullptr);
    vehOfSlot[s] = v;
    return s;
}

// one step of the emulated engine, fed with what the restatement spawned in its own (already executed) step
void deviceStep(Oracle &o) {
    HostSim &H = *S;
    View &V = H.V;
    Routing &R = *o.routing;
    // ---- host part: spawn records (HostEngine::prepareStep), lane-sorted, stable ----
    std::vector<SpawnRec> recs;
    for (Veh *v : o.spawnedThisStep) {
        const int s = newSlot(v);
        const int route = R.intern(v->route);
        if (R.route(route).roads != v->route) { printf("probe: interning the resolved route changed it (prio %d)\n", v->priority); ++g_fail; }
        SpawnRec r{};
        r.slot = s; r.lane = v->firstLaneForProbe; r.tmpl = s; r.priority = v->priority;
        r.plan = R.lanePlan(route, 0, o.net.laneIdx[r.lane]);
        recs.push_back(r);
        H.tmpl[s] = toDevice(v->t, o.interval);
        H.tmpl[s].speed0 = v->initialSpeedForProbe;
    }
    std::stable_sort(recs.begin(), recs.end(), [](const SpawnRec &a, const SpawnRec &b) { return a.lane < b.lane; });
    H.setPlans(R);   // (routes are interned lazily: tables may have grown)
    H.spawn[0].slot = (int) recs.size();
    for (size_t k = 0; k < recs.size(); ++k) H.spawn[k + 1] = recs[k];
    V.spawn = H.spawn.p() + 1;
    V.par = (int) (H.steps & 1);
    const int G = 3;   // blocks per launch: more than one, so the grid-stride loops are exercised
    H.run(G, [&](int b, int n) { phase_ingest(V, b, n); });
    if (V.lcOn) {
        for (int k = 0; k < 64; ++k) H.spare[k] = g_nextSlot + k;   // slots lent for this step's shadows
        V.lc.nSpare = 64;
        H.lcCtrl.nCand = H.lcCtrl.nInvolved = H.lcCtrl.nShadows = H.lcCtrl.spareUsed = 0;   // k_lc_begin
        H.run(G, [&](int, int) { k_lc_admitted(V, V.lc); });
        H.run(G, [&](int, int) { k_lc_segments(V, V.lc); });
        H.run(G, [&](int, int) { k_lc_signal(V, V.lc); });
        if (const char *tp = getenv("PROBE_TRACE_PRIO")) {
            const int want = atoi(tp);
            for (auto &kv : o.pool) if (kv.first == want && slotOf.count(kv.second)) {
                const int s = slotOf.at(kv.second), p = H.pos[s];
                if (p < 0) continue;
                const LcSlot &L = H.lcSlot[s];
                const int dd = H.L.posDrv[p];
                const int rp = lcRoadPos(V, V.lc, L.plan, H.nav[p].x);
                printf("  signal step %zu: drivable %d laneIdx %d/%d dis %.4f own gap %.6f len %.2f seg %d plan %d planIdx %d roadPos %d next %d -> target %d epoch %d\n", o.step, dd, H.L.laneIdx[dd],
                       H.L.laneRoadN[dd], H.kin[p].x, L.gap, H.tmpl[H.ids[p].y].len, H.segIdx[p], L.plan, H.nav[p].x, rp, H.ids[p].w, L.sendTarget, L.sendEpoch);
                {
                    Veh *v = kv.second;
                    printf("    restatement: iCur %d route size %zu onLastRoad %d; routerNextOf(outer) %d; plan's route %d roads:", v->iCur, v->route.size(), (int) o.onLastRoad(*v),
                           dd + 1 < V.nLanes ? o.routerNextOf(*v, dd + 1) : -9, H.lanePlans.planRoute[L.plan]);
                    for (int r2 : v->route) printf(" %d", r2);
                    printf(" | lane road %d; lanePlan ids for roadPos %d:", o.net.laneRoad[dd], rp);
                    for (int k2 = 0; k2 < H.L.laneRoadN[dd]; ++k2) { const int np = lcLanePlan(V.lc, L.plan, rp, dd - H.L.laneIdx[dd] + k2); printf(" %d(next %d)", np, H.plans.planData[H.plans.planBeg[np] + 1]); }
                    printf("\n");
                }
                for (int adj : {dd + 1, dd - 1}) {
                    if (adj < 0 || adj >= V.nLanes || o.net.laneRoad[adj] != o.net.laneRoad[dd]) continue;
                    const int lp = lcVehicleAfter(V, V.lc, adj, H.kin[p].x, H.segIdx[p]);
                    printf("    lane %d: continues %d, vehicle ahead pos %d est %.4f (count %d)\n", adj, (int) lcLaneContinues(V, V.lc, L.plan, rp, adj, H.ids[p].w == -1), lp,
                           lp < 0 ? H.L.drvLength[adj] - H.kin[p].x : H.kin[lp].x - H.kin[p].x - H.tmpl[H.ids[lp].y].len, H.count[adj]);
                }
            }
        }
        if (getenv("CITYFLOW_B200_LC_SERIAL")) H.run(1, [&](int, int) { k_lc_schedule(V, V.lc); });
        else {   // the per-road form DeviceSim launches by default
            H.run(1, [&](int, int) { k_lc_order(V, V.lc); });
            H.run(G, [&](int, int) { k_lc_schedule_roads(V, V.lc); });
            H.run(1, [&](int, int) { k_lc_log(V, V.lc); });
        }
        // host round trip: the shadows' priorities, in schedule order (HostEngine::nextStepLaneChange); here they
        // come from the restatement's own draws, matched by parent
        const int ns = H.lcCtrl.nShadows;
        for (int k = 0; k < ns; ++k) {
            Veh *parent = vehOfSlot[H.shadowLog[k].x];
            int pr = INT_MIN;
            for (auto &sp : o.shadowsThisStep) if (sp.first == parent) pr = sp.second;
            CHECK(pr != INT_MIN, "the device created a shadow for prio %d, the restatement did not", parent ? parent->priority : 0);
            H.prio[k] = pr;
            // the restatement's shadow object, if it survived its first step (it may have aborted at once)
            auto it = pr != INT_MIN ? o.pool.find(pr) : o.pool.end();
            if (it != o.pool.end()) {
                const int sh = H.shadowLog[k].y;
                slotOf[it->second] = sh;
                if ((int) vehOfSlot.size() <= sh) vehOfSlot.resize(sh + 1, nullptr);
                vehOfSlot[sh] = it->second;
            }
        }
        CHECK(ns == (int) o.shadowsThisStep.size(), "shadows created: restatement %zu, device %d", o.shadowsThisStep.size(), ns);
        for (auto &sp : o.shadowsThisStep) {   // diagnostics: a parent the device did not serve
            Veh *pv = sp.first;
            const int ps = slotOf.at(pv);
            bool found = false;
            for (int k = 0; k < ns; ++k) found |= H.shadowLog[k].x == ps;
            if (!found) {
                const LcSlot &L = H.lcSlot[ps];
                const int p = H.pos[ps];
                printf("  missing shadow of prio %d: device send valid %d target %d (restatement target %d) recv valid %d tgtL %d tgtF %d gaps %g %g | stale gap %g vs %g | dis %g seg %d | cand %d\n",
                       pv->priority, (int) lcSendValid(L, (int) o.step), L.sendTarget, pv->sigSend ? pv->sigSend->target : -9, (int) lcRecvValid(L, (int) o.step), L.tgtLeader, L.tgtFollower,
                       L.leaderGap, L.followerGap, L.gap, pv->gap, H.kin[p].x, H.segIdx[p], H.lcCtrl.nCand);
            }
        }
        g_nextSlot += H.lcCtrl.spareUsed;
        g_shadows += ns;
        if (ns > 0) H.run(1, [&](int, int) { k_lc_priorities(V, V.lc, H.prio.p(), ns); });
        H.run(G, [&](int, int) { k_lc_leader(V, V.lc); });
        if (const char *tp = getenv("PROBE_TRACE_PRIO")) {
            const int want = atoi(tp);
            for (int k = 0; k < ns; ++k) if (H.prio[k] == want) {
                const int sh = H.shadowLog[k].y, p = H.pos[sh];
                printf("  mid-step: shadow slot %d at pos %d (drivable %d, count %d) next %d planIdx %d leader %d V.gap %.6f own %.6f; nAct %d; parent tgtLeader %d\n", sh, p, H.L.posDrv[p],
                       H.count[H.L.posDrv[p]], H.ids[p].w, H.nav[p].x, H.leader[p], H.gap[p], H.lcSlot[sh].gap, H.ctrl.nAct[V.par], H.lcSlot[H.shadowLog[k].x].tgtLeader);
                bool inAct = false;
                for (int a2 = 0; a2 < H.ctrl.nAct[V.par]; ++a2) inAct |= V.actList[V.par][a2] == H.L.posDrv[p];
                printf("  drivable in actList: %d\n", (int) inAct);
            }
        }
    }
    H.run(G, [&](int b, int n) { phase_notify(V, b, n); });
    H.run(G, [&](int b, int n) { phase_control(V, b, n); });
    if (V.lcOn) {
        if (getenv("CITYFLOW_B200_LC_SERIAL")) H.run(1, [&](int, int) { k_lc_control_tail(V, V.lc); });
        else {
            H.run(1, [&](int, int) { k_lc_tail_order(V, V.lc); });
            H.run(G, [&](int, int) { k_lc_tail_roads(V, V.lc); });
            H.run(1, [&](int, int) { k_lc_tail_clear(V, V.lc); });
        }
    }
    H.run(G, [&](int b, int n) { phase_move(V, b, n); });
    H.run(G, [&](int b, int n) { phase_leader(V, b, n); });
    H.steps += 1;
    CHECK(H.ctrl.error == 0 && H.lcCtrl.error == 0, "device error flags %d / %d", H.ctrl.error, H.lcCtrl.error);
}

void compare(Oracle &o, std::vector<Veh *> &removedThisStep) {
    HostSim &H = *S;
    View &V = H.V;
    // shadows created this step: map the restatement's object to the device's slot (through the parent)
    for (auto &kv : o.pool) {
        Veh *v = kv.second;
        if (!v->running || slotOf.count(v)) continue;
        CHECK(v->partnerType == 2 && v->partner && slotOf.count(v->partner), "unknown running vehicle prio %d", v->priority);
        if (v->partner && slotOf.count(v->partner)) {
            const int sh = H.lcSlot[slotOf.at(v->partner)].partner;
            CHECK(sh >= 0, "parent prio %d has no shadow on the device", v->partner->priority);
            if (sh >= 0) { slotOf[v] = sh; if ((int) vehOfSlot.size() <= sh) vehOfSlot.resize(sh + 1, nullptr); vehOfSlot[sh] = v; }
        }
    }
    if (const char *tp = getenv("PROBE_TRACE_PRIO")) {
        const int want = atoi(tp);
        for (auto &kv : o.pool) if (kv.first == want && kv.second->running && slotOf.count(kv.second)) {
            Veh *v = kv.second; const int s = slotOf.at(v); const LcSlot &L = H.lcSlot[s]; const int p = H.pos[s];
            printf("  trace step %zu prio %d: type %d/%d drivable %d/%d dis %.4f/%.4f leader %d/%d own gap %.6f/%.6f V.gap %.6f changing %d/%d\n", o.step, want, v->partnerType, L.type,
                   v->drivable, H.L.posDrv[p], v->dis, H.kin[p].x, v->leader ? v->leader->priority : 0, H.leader[p] >= 0 ? H.ids[H.leader[p]].z : 0, v->gap, L.gap, H.gap[p], v->changing, L.changing);
        }
    }
    CHECK((int) o.activeCount == H.ctrl.active, "active vehicles %zu vs %d", o.activeCount, H.ctrl.active);
    for (int d = 0; d < V.nDrv; ++d) {
        CHECK((int) o.lists[d].size() == H.count[d], "drivable %d holds %zu vs %d vehicles", d, o.lists[d].size(), H.count[d]);
        if ((int) o.lists[d].size() != H.count[d]) continue;
        int k = 0;
        for (Veh *v : o.lists[d]) {
            const int p = H.L.off[d] + k++;
            const int s = slotOf.count(v) ? slotOf.at(v) : -1;
            CHECK(H.ids[p].x == s, "drivable %d position %d: slot %d, expected %d (prio %d)", d, k - 1, H.ids[p].x, s, v->priority);
            if (H.ids[p].x != s) continue;
            CHECK(H.pos[s] == p && H.ids[p].z == v->priority, "prio %d: pos / priority record", v->priority);
            CHECK(H.kin[p].x == v->dis && H.kin[p].y == v->t.speed, "prio %d: dis %.17g/%.17g speed %.17g/%.17g", v->priority, v->dis, H.kin[p].x,
                  v->t.speed, H.kin[p].y);
            const int lp = H.leader[p];
            CHECK((v->leader ? slotOf.at(v->leader) : -1) == (lp >= 0 ? H.ids[lp].x : -1), "prio %d: leader", v->priority);
            if (v->leader && lp >= 0) CHECK(H.gap[p] == v->gap, "prio %d: gap %.17g vs %.17g", v->priority, v->gap, H.gap[p]);
            int devBlocker = H.nav[p].z;   // a blocker that left in the step just done is dropped lazily on the device (DeviceSim::debugDump)
            if (devBlocker >= 0 && H.delStep[devBlocker] == H.ctrl.step - 1) devBlocker = -1;
            CHECK((v->blocker ? slotOf.at(v->blocker) : -1) == devBlocker, "prio %d (type %d) on drivable %d: blocker %d (prio %d) vs slot %d", v->priority,
                  v->partnerType, d, v->blocker ? slotOf.at(v->blocker) : -1, v->blocker ? v->blocker->priority : 0, devBlocker);
            CHECK((int) v->enterLaneLinkTime == H.nav[p].w && v->prevDrivable == H.nav[p].y, "prio %d: enterLaneLinkTime / prevDrivable", v->priority);
            if (V.lcOn) {
                const LcSlot &L = H.lcSlot[s];
                CHECK(L.type == v->partnerType && (v->partner ? slotOf.at(v->partner) : -1) == L.partner, "prio %d: partner type %d/%d", v->priority, v->partnerType, L.type);
                CHECK(L.gap == v->gap, "prio %d (drivable %d, list index %d of %d, leader %d): the vehicle's own gap value %.17g vs %.17g", v->priority, d, k - 1,
                      H.count[d], v->leader ? v->leader->priority : 0, v->gap, L.gap);
                CHECK(L.changing == (int) v->changing && L.offset == v->offset, "prio %d: changing %d/%d offset %g/%g", v->priority, v->changing, L.changing, v->offset, L.offset);
                CHECK(L.waiting == v->waitingTime && L.lastChange == v->lastChangeTime && L.lastDir == v->lastDir, "prio %d: waiting %g/%g lastChange %g/%g lastDir %d/%d",
                      v->priority, v->waitingTime, L.waiting, v->lastChangeTime, L.lastChange, v->lastDir, L.lastDir);
            }
            ++g_checked;
        }
    }
    // waiting queues
    for (int l = 0; l < V.nLanes; ++l) {
        int n = 0;
        for (int s = H.waitHead[l]; s >= 0; s = H.waitNext[s]) ++n;
        CHECK(n == (int) o.waiting[l].size(), "lane %d: waiting queue %zu vs %d", l, o.waiting[l].size(), n);
    }
    // finished ring (HostEngine::drain)
    int fin = 0;
    for (int k = 0; k < H.ctrl.finCount; ++k) {
        const int tag = H.finSlots[k].x, s = tag & ~0x40000000;
        if (!(tag & 0x40000000)) ++fin;
        Veh *v = vehOfSlot[s];
        if (v) { slotOf.erase(v); vehOfSlot[s] = nullptr; }
    }
    H.ctrl.finCount = 0;
    g_finished += fin;
    CHECK(g_finished == o.finishedCnt, "finished vehicles %d vs %lld", o.finishedCnt, g_finished);
    (void) removedThisStep;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) { fprintf(stderr, "usage: device_step_probe config.json steps\n"); return 64; }
    Oracle o;
    if (!o.load(argv[1])) { fprintf(stderr, "cannot load %s\n", argv[1]); return 2; }
    o.routing->enableLanePlans();
    HostSim H;
    std::vector<cfb::VehicleTemplate> fleet;
    for (const auto &f : o.flows) fleet.push_back(f.def.tmpl);
    H.init(o.net, o.interval, o.rlTrafficLight, o.laneChange, cfb::bucketSpacing(fleet));
    S = &H;
    const int steps = atoi(argv[2]);
    std::vector<Veh *> removed;
    for (int s = 0; s < steps && g_fail == 0; ++s) {
        o.nextStep();
        deviceStep(o);
        compare(o, removed);
    }
    printf("%s %lld steps, %lld vehicle states, %lld finished, %lld shadows, %d failures\n", g_fail ? "FAIL" : "OK", H.steps, g_checked, g_finished, g_shadows, g_fail);
    return g_fail ? 1 : 0;
}
