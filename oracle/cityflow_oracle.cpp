// TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's Engine::nextStep hot path.
//
// This file is the executable specification the CUDA kernels are checked against.  It is a
// single-threaded, plain C++ restatement (vectors instead of the reference's pointer graph) of
//   Engine::nextStep          engine.cpp:566-594   and the phase functions it calls
//   Flow::nextStep            flow.cpp:6-22        Vehicle ctor vehicle.cpp:38-47
//   Engine::planRoute/handleWaiting/threadNotifyCross/vehicleControl/updateLocation/
//   threadUpdateAction/threadUpdateLeaderAndGap   engine.cpp:188-251, 282-372, 402-516
//   Vehicle::*                vehicle.cpp:49-73, 107-143, 157-376
//   Router lookahead          router.cpp:23-129
//   Cross::canPass/notify     roadnet.cpp:595-676   Lane::available/canEnter roadnet.cpp:428-445
//   TrafficLight::passTime    trafficlight.cpp:29-37
// Every function cites the reference lines it follows.
//
// laneChange=true (lanechange.cpp, engine.cpp:195-244, 374-400, 792-820, roadnet.cpp:837-898) IS
// restated, but the unmodified reference cannot pin it: there the order in which lane-change
// candidates are scheduled is the heap-address order of a std::set<Vehicle*> and one input of the
// decision (ControllerInfo::gap of a vehicle that never had a leader) is read uninitialised.  The
// pin is the reference built with those two things defined (oracle/lc_order_patch.sh: set ordered
// by priority, gap = 0) -- oracle/_ref/refdump_lcorder, single worker thread.
//
// PARITY PINNING: tests/test_oracle_vs_ref.py runs this oracle and the compiled, unmodified
// reference (oracle/_ref, built by oracle/Makefile) side by side and requires bit-equal
// per-vehicle (drivable, dis, speed, leader, gap, blocker) and per-lane counts every step; the
// committed fixtures in tests/golden/ were generated from the compiled reference by
// tests/golden/make_golden.py.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may use this file.  The
// product (cityflow_b200/) never links or calls it.  It reuses the product's *static* loaders
// (roadnet.cpp / flows.cpp, themselves pinned against `refdump static`) for file parsing only.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <iostream>
#include <map>
#include <memory>
#include <random>
#include <set>
#include <string>
#include <vector>

#include "../cityflow_b200/csrc/flows.h"
#include "../cityflow_b200/csrc/json_min.h"
#include "../cityflow_b200/csrc/roadnet.h"

namespace {

using cfb::RoadNet;
using cfb::VehicleTemplate;

constexpr double kEps = 1e-8;  // utility.h:15
inline double max2(double x, double y) { return x > y ? x : y; }  // utility.h:66
inline double min2(double x, double y) { return x < y ? x : y; }  // utility.h:70

struct Veh {
    VehicleTemplate t;
    int priority = 0, flow = -1, cnt = -1;
    double enterTime = 0;
    // ControllerInfo (vehicle.h:81-95)
    double dis = 0;
    int drivable = -1, prevDrivable = -1;
    double approachDist = 0, gap = 0;
    int64_t enterLaneLinkTime = INT_MAX;
    Veh *leader = nullptr, *blocker = nullptr;
    bool running = false;
    // Router (router.h:22-28)
    std::vector<int> route;
    int iCur = 0;
    std::deque<int> planned;
    bool routeValid = false;
    // Buffer (vehicle.h:54-72)
    bool bDisSet = false, bSpeedSet = false, bDrvSet = false, bEndSet = false, bBlockerSet = false,
         bEnterSet = false, bCustomSet = false;
    double bDis = 0, bDelta = 0, bSpeed = 0, bCustom = 0;
    int bDrv = -1;
    bool bEnd = false;
    Veh *bBlocker = nullptr;
    int64_t bEnter = 0;
    // LaneChangeInfo (vehicle.h:74-79)
    int partnerType = 0;             // 0 none, 1 = has a shadow, 2 = is a shadow
    Veh *partner = nullptr;
    double offset = 0;
    size_t segIndex = 0;
    // LaneChange / SimpleLaneChange state (lanechange.h:15-44)
    struct Signal {                  // lanechange.h:17-24 (value-initialised by make_shared: all zero)
        int urgency = 0, direction = 0;
        int target = -1;             // lane id
        Veh *source = nullptr;
    };
    std::shared_ptr<Signal> sigRecv, sigSend;
    int lastDir = 0;
    Veh *targetLeader = nullptr, *targetFollower = nullptr;
    double leaderGap = 0, followerGap = 0, waitingTime = 0;
    bool changing = false, lcFinished = false;
    double lastChangeTime = 0;
    double ctlHead = 0;              // device form: order-independent part of the next speed
    int firstLaneForProbe = -1;      // tests/device_step_probe.cpp: the lane whose waiting queue the vehicle joined
    double initialSpeedForProbe = 0; //                               VehicleInfo::speed at creation
    bool isReal() const { return partnerType != 2; }                                   // vehicle.h:278
    bool planChange() const { return (sigSend && sigSend->target >= 0 && sigSend->target != drivable) || changing; }  // lanechange.cpp:23-25
};

struct FlowState {
    cfb::FlowDef def;
    double nowTime = 0, currentTime = 0;
    int cnt = 0;
    bool valid = true;
};

struct Oracle {
    RoadNet net;
    std::vector<FlowState> flows;
    double interval = 1.0;
    bool rlTrafficLight = false;
    int seed = 0;
    std::mt19937 rnd;
    size_t step = 0;
    size_t activeCount = 0;
    int manuallyPushCnt = 0;
    int finishedCnt = 0;
    double cumulativeTravelTime = 0;
    std::map<int, Veh *> pool;                       // vehiclePool keyed by priority (engine.h:25)
    std::vector<std::vector<Veh *>> lists;           // per drivable, front -> back
    std::vector<std::deque<Veh *>> waiting;          // per lane
    std::vector<std::vector<Veh *>> planRouteBuffer; // per road
    std::vector<Veh *> notifyVeh[2];                 // per cross
    std::vector<double> notifyDist[2];
    std::vector<int> curPhase;
    std::vector<double> remain;
    std::vector<std::pair<Veh *, double>> pushBuffer;
    std::set<Veh *> removeBuffer;
    // laneChange=true (restated against the reference built with the priority-ordered worker set,
    // oracle/lc_order_patch.sh): segment index per lane (roadnet.cpp:687-691, :852-875)
    bool laneChange = false;
    // "Device form" (DESIGN.md section 10): the same step computed in the decomposition planned for the
    // GPU -- order-independent work in arbitrary order, per-road scheduling, only the few vehicles
    // involved in a lane change processed in priority order.  Must give identical states; exists to
    // check that decomposition on the CPU (tests/test_cpu.py).
    bool deviceForm = false;
    std::vector<std::vector<double>> segStart;            // [lane][segment] startPos
    std::vector<std::vector<std::vector<Veh *>>> segVeh;  // [lane][segment] vehicles, list order
    int ties = 0;  // pushBuffer ties (same target drivable, equal dis): order unspecified in the reference
    int maxRefusedCross = -1;  // highest index in its laneLink's cross list at which Cross::canPass refused a vehicle
    cfb::Routing *routing = nullptr;

    int nLanes() const { return net.nLanes(); }
    bool isLink(int d) const { return d >= net.nLanes(); }
    double drvLength(int d) const { return isLink(d) ? net.llLength[d - nLanes()] : net.laneLength[d]; }
    double drvMaxSpeed(int d) const { return isLink(d) ? 10000 : net.laneMaxSpeed[d]; }  // roadnet.h:456
    Veh *lastVeh(int d) const { return lists[d].empty() ? nullptr : lists[d].back(); }
    Veh *firstVeh(int d) const { return lists[d].empty() ? nullptr : lists[d].front(); }
    bool linkAvailable(int ll) const {  // RoadLink::isAvailable, roadnet.h:429-431
        int rl = net.llRoadLink[ll], in = net.rlInter[rl];
        int ph = net.interPhaseBeg[in] + curPhase[in];
        return net.phaseAvail[net.phaseAvailBeg[ph] + (rl - net.interRoadLinkBeg[in])] != 0;
    }
    double currentTime() const { return step * interval; }  // engine.cpp:678

    // ---------------- Router ----------------
    // Router::getNextDrivable(const Drivable*) router.cpp:49-76
    int routerNextOf(const Veh &v, int cur) const {
        if (isLink(cur)) return net.llEndLane[cur - nLanes()];
        int road = net.laneRoad[cur];
        int r = v.iCur;
        while (r < (int) v.route.size() && v.route[r] != road) ++r;
        int ll = routing->chooseLink(cur, v.route, r);  // selectLaneLink rule, router.cpp:96-129
        return ll < 0 ? -1 : nLanes() + ll;
    }
    // Router::getNextDrivable(size_t i) router.cpp:39-47
    int nextDrivable(Veh &v, size_t i = 0) const {
        while (i >= v.planned.size()) {
            int from = v.planned.empty() ? v.drivable : v.planned.back();
            if (from < 0) return -1;
            v.planned.push_back(routerNextOf(v, from));
        }
        return v.planned[i];
    }
    // Router::update router.cpp:78-94
    void routerUpdate(Veh &v) const {
        if (!isLink(v.drivable)) {
            int road = net.laneRoad[v.drivable];
            while (v.iCur < (int) v.route.size() && v.route[v.iCur] != road) ++v.iCur;
        }
        while (!v.planned.empty()) {
            int d = v.planned.front();
            v.planned.pop_front();
            if (d == v.drivable) break;
        }
    }

    // ---------------- Vehicle dynamics ----------------
    // vehicle.cpp:200-209
    static double noCollisionSpeed(double vL, double dL, double vF, double dF, double gap, double dt, double targetGap) {
        double c = vF * dt / 2 + targetGap - 0.5 * vL * vL / dL - gap;
        double a = 0.5 / dF;
        double b = 0.5 * dt;
        if (b * b < 4 * a * c) return -100;
        double v1 = 0.5 / a * (sqrt(b * b - 4 * a * c) - b);
        double v2 = 2 * vL - dL * dt + 2 * (gap - targetGap) / dt;
        return min2(v1, v2);
    }
    // vehicle.cpp:212-238
    double carFollowSpeed(const Veh &v) const {
        const Veh *L = v.leader;
        if (!L) return v.bCustomSet ? v.bCustom : v.t.maxSpeed;
        double s = noCollisionSpeed(L->t.speed, L->t.maxNegAcc, v.t.speed, v.t.maxNegAcc, v.gap, interval, 0);
        if (v.bCustomSet) return min2(v.bCustom, s);
        double assumeDecel = 0, leaderSpeed = L->t.speed;
        if (v.t.speed > leaderSpeed) assumeDecel = v.t.speed - leaderSpeed;
        s = min2(s, noCollisionSpeed(L->t.speed, L->t.usualNegAcc, v.t.speed, v.t.usualNegAcc, v.gap, interval, v.t.minGap));
        s = min2(s, (v.gap + (leaderSpeed + assumeDecel / 2) * interval - v.t.speed * interval / 2) /
                        (v.t.headwayTime + interval / 2));
        return s;
    }
    static double minBrakeDistance(const Veh &v) { return 0.5 * v.t.speed * v.t.speed / v.t.maxNegAcc; }  // vehicle.h:239
    // vehicle.cpp:302-306
    static double brakeDistanceAfterAccel(const Veh &v, double acc, double dec, double dt) {
        double cur = v.t.speed;
        double next = cur + acc * dt;
        return (cur + next) * dt / 2 + (next * next / dec / 2);
    }
    // vehicle.cpp:240-250
    double stopBeforeSpeed(const Veh &v, double distance) const {
        if (brakeDistanceAfterAccel(v, v.t.usualPosAcc, v.t.usualNegAcc, interval) < distance)
            return v.t.speed + v.t.usualPosAcc * interval;
        double takeInterval = 2 * distance / (v.t.speed + kEps) / interval;
        if (takeInterval >= 1) return v.t.speed - v.t.speed / (int) takeInterval;
        return v.t.speed - v.t.speed / takeInterval;
    }
    // vehicle.cpp:275-282
    double distanceUntilSpeed(const Veh &v, double speed, double acc) const {
        if (speed <= v.t.speed) return 0;
        int stage1steps = std::floor((speed - v.t.speed) / acc / interval);
        double stage1speed = v.t.speed + stage1steps * acc / interval;
        double stage1dis = (v.t.speed + stage1speed) * (stage1steps * interval) / 2;
        return stage1dis + (stage1speed < speed ? ((stage1speed + speed) * interval / 2) : 0);
    }
    // vehicle.cpp:252-268
    int reachSteps(const Veh &v, double distance, double targetSpeed, double acc) const {
        if (distance <= 0) return 0;
        if (v.t.speed > targetSpeed) return std::ceil(distance / v.t.speed);
        double du = distanceUntilSpeed(v, targetSpeed, acc);
        if (du > distance)
            return std::ceil((std::sqrt(v.t.speed * v.t.speed + 2 * acc * distance) - v.t.speed) / acc / interval);
        return std::ceil((targetSpeed - v.t.speed) / acc / interval) + std::ceil((distance - du) / targetSpeed / interval);
    }
    // vehicle.cpp:270-273
    int reachStepsOnLaneLink(const Veh &v, double distance, int ll) const {
        return reachSteps(v, distance, net.linkIsTurn(ll) ? v.t.turnSpeed : v.t.maxSpeed, v.t.usualPosAcc);
    }
    // vehicle.cpp:284-287
    static bool canYield(const Veh &v, double dist) {
        return (dist > 0 && minBrakeDistance(v) < dist - v.t.yieldDistance) || (dist < 0 && dist + v.t.len < 0);
    }
    // Lane::canEnter roadnet.cpp:437-445
    bool laneCanEnter(int lane, const Veh &v) const {
        const Veh *tail = lastVeh(lane);
        if (!tail) return true;
        return tail->dis > tail->t.len + v.t.len || tail->t.speed >= 2;
    }
    // Cross::canPass roadnet.cpp:603-676
    bool canPass(int cross, const Veh &v, int ll, double distanceToLaneLinkStart) const {
        int i = (net.crossLink[0][cross] == ll) ? 0 : 1;
        Veh *foe = notifyVeh[1 - i][cross];
        int t1 = net.rlType[net.llRoadLink[net.crossLink[i][cross]]];
        int t2 = net.rlType[net.llRoadLink[net.crossLink[1 - i][cross]]];
        double d1 = net.crossDist[i][cross] - distanceToLaneLinkStart, d2 = notifyDist[1 - i][cross];
        if (!foe) return true;
        if (!canYield(v, d1)) return true;
        int yield = 0;
        if (!canYield(*foe, d2)) yield = 1;
        if (yield == 0) {
            if (t1 > t2) {
                yield = -1;
            } else if (t1 < t2) {
                if (d2 > 0) {
                    int foeSteps = reachStepsOnLaneLink(*foe, d2, net.crossLink[1 - i][cross]);
                    int mySteps = reachStepsOnLaneLink(v, d1, net.crossLink[i][cross]);
                    if (foeSteps > mySteps) yield = -1;
                } else {
                    if (d2 + foe->t.len < 0) yield = -1;
                }
                if (yield == 0) yield = 1;
            } else {
                if (d2 > 0) {
                    int foeSteps = reachStepsOnLaneLink(*foe, d2, net.crossLink[1 - i][cross]);
                    int mySteps = reachStepsOnLaneLink(v, d1, net.crossLink[i][cross]);
                    if (foeSteps > mySteps) yield = -1;
                    else if (foeSteps < mySteps) yield = 1;
                    else {
                        double e1 = (double) (size_t) v.enterLaneLinkTime, e2 = (double) (size_t) foe->enterLaneLinkTime;
                        if (e1 == e2) {
                            if (d1 == d2) yield = v.priority > foe->priority ? -1 : 1;
                            else yield = d1 < d2 ? -1 : 1;
                        } else {
                            yield = e1 < e2 ? -1 : 1;
                        }
                    }
                } else {
                    yield = d2 + foe->t.len < 0 ? -1 : 1;
                }
            }
        }
        if (yield == 1) {  // deadlock detection over committed blockers (Floyd), roadnet.cpp:662-674
            Veh *fast = foe, *slow = foe;
            while (fast != nullptr && fast->blocker != nullptr) {
                slow = slow->blocker;
                fast = fast->blocker->blocker;
                if (slow == fast) { yield = -1; break; }
            }
        }
        return yield == -1;
    }
    // vehicle.cpp:289-300
    bool isIntersectionRelated(Veh &v) const {
        if (isLink(v.drivable)) return true;
        int nd = nextDrivable(v);
        return nd >= 0 && isLink(nd) && drvLength(v.drivable) - v.dis <= v.approachDist;
    }
    // vehicle.cpp:337-376
    double intersectionRelatedSpeed(Veh &v) {
        double s = v.t.maxSpeed;
        int nd = nextDrivable(v);
        int ll = -1;
        if (nd >= 0 && isLink(nd)) {
            ll = nd - nLanes();
            if (!linkAvailable(ll) || !laneCanEnter(net.llEndLane[ll], v)) {
                if (minBrakeDistance(v) > drvLength(v.drivable) - v.dis) {
                    // cannot brake before the line: falls through
                } else {
                    s = min2(s, stopBeforeSpeed(v, drvLength(v.drivable) - v.dis));
                    return s;
                }
            }
            if (net.linkIsTurn(ll)) s = min2(s, v.t.turnSpeed);
        }
        if (ll < 0 && isLink(v.drivable)) ll = v.drivable - nLanes();
        double distanceToLaneLinkStart = !isLink(v.drivable) ? -(drvLength(v.drivable) - v.dis) : v.dis;
        for (size_t ci = 0; ci < net.llCrosses[ll].size(); ++ci) {
            const cfb::CrossRef &cr = net.llCrosses[ll][ci];
            double distanceOnLaneLink = net.crossDist[cr.side][cr.cross];
            if (distanceOnLaneLink < distanceToLaneLinkStart) continue;
            if (!canPass(cr.cross, v, ll, distanceToLaneLinkStart)) {
                maxRefusedCross = std::max(maxRefusedCross, (int) ci);
                s = min2(s, stopBeforeSpeed(v, distanceOnLaneLink - distanceToLaneLinkStart - v.t.yieldDistance));
                v.bBlocker = notifyVeh[1 - cr.side][cr.cross];  // setBlocker(getFoeVehicle)
                v.bBlockerSet = true;
                break;
            }
        }
        return s;
    }
    // vehicle.cpp:308-335 (laneChange off)
    // The part of getNextSpeed that reads only state committed before the phase (and buffers only
    // the vehicle's own blocker): independent of the order vehicles are processed in.
    double nextSpeedHead(Veh &v) {
        double s = v.t.maxSpeed;
        s = min2(s, v.t.speed + v.t.maxPosAcc * interval);
        s = min2(s, drvMaxSpeed(v.drivable));
        s = min2(s, carFollowSpeed(v));
        if (isIntersectionRelated(v)) s = min2(s, intersectionRelatedSpeed(v));
        return s;
    }
    double nextSpeed(Veh &v) {
        double s;
        if (deviceForm) { s = v.ctlHead; }   // computed by controlDeviceForm()'s first pass
        else s = nextSpeedHead(v);
        {   // vehicle.cpp:323-329.  `if (laneChange)` there tests the vehicle's LaneChange OBJECT (always
            // present), not the engine's laneChange option: the block also runs with laneChange=false.
            // Without signals the yield term is 100 (no effect below 100 m/s); the second term makes a
            // vehicle whose lane cannot continue its route stop at the end of the lane -- reachable on
            // networks where a first lane links to the next road only through lanes that cannot reach
            // the road after it (router.cpp:23-37 vs :65-73).
            s = min2(s, yieldSpeed(v));
            if (!onValidLane(v)) {
                double vn = noCollisionSpeed(0, 1, v.t.speed, v.t.maxNegAcc, drvLength(v.drivable) - v.dis, interval, v.t.minGap);
                s = min2(s, vn);
            }
        }
        s = max2(s, v.t.speed - v.t.maxNegAcc * interval);
        return s;
    }

    // ---------------- lane change (lanechange.cpp, engine.cpp:195-244, 374-400, 792-820) ----------------
    bool isLastRoad(const Veh &v, int d) const { return !isLink(d) && net.laneRoad[d] == v.route.back(); }   // router.cpp:131-134
    bool onLastRoad(const Veh &v) const { return isLastRoad(v, v.drivable); }                                  // router.cpp:136-138
    bool onValidLane(Veh &v) const { return !(nextDrivable(v) < 0 && !onLastRoad(v)); }                        // router.h:66-68
    int innerLane(int l) const { return net.laneIdx[l] > 0 ? l - 1 : -1; }                                     // roadnet.h:335-337
    int outerLane(int l) const { return net.laneIdx[l] < net.roadNumLanes(net.laneRoad[l]) - 1 ? l + 1 : -1; } // roadnet.h:339-342
    // Lane::initSegments roadnet.cpp:863-875
    void initSegments() {
        if (deviceForm) {  // no segment lists: segmentIndex(p) = min(natural segment of p, segmentIndex(p-1)), a prefix-min
            for (int l = 0; l < nLanes(); ++l) {
                int run = (int) segStart[l].size() - 1;
                for (Veh *v : lists[l]) {
                    int nat = (int) segStart[l].size() - 1;
                    while (nat > 0 && !(v->dis >= segStart[l][nat])) --nat;   // highest i with dis >= startPos(i); segment 0 starts at 0
                    if (!(v->dis >= segStart[l][nat])) nat = -1;              // (dis < 0 cannot happen; the reference would skip the vehicle)
                    run = std::min(run, nat);
                    if (run >= 0) v->segIndex = (size_t) run;
                }
            }
            return;
        }
        for (int l = 0; l < nLanes(); ++l) {
            auto it = lists[l].begin(), end = lists[l].end();
            for (int i = (int) segStart[l].size() - 1; i >= 0; --i) {
                auto &sv = segVeh[l][i];
                sv.clear();
                while (it != end && (*it)->dis >= segStart[l][i]) {
                    sv.push_back(*it);
                    (*it)->segIndex = (size_t) i;
                    ++it;
                }
            }
        }
    }
    // Lane::getVehicleBeforeDistance roadnet.cpp:877-887
    Veh *vehicleBefore(int lane, double dis, size_t segIndex) const {
        if (deviceForm) {  // the segment lists are the list filtered by segmentIndex
            for (int i = (int) segIndex; i >= 0; --i)
                for (Veh *v : lists[lane])
                    if ((int) v->segIndex == i && v->dis < dis) return v;
            return nullptr;
        }
        for (int i = (int) segIndex; i >= 0; --i)
            for (Veh *v : segVeh[lane][i])
                if (v->dis < dis) return v;
        return nullptr;
    }
    // Lane::getVehicleAfterDistance roadnet.cpp:889-898
    Veh *vehicleAfter(int lane, double dis, size_t segIndex) const {
        if (deviceForm) {
            for (size_t i = segIndex; i < segStart[lane].size(); ++i)
                for (auto it = lists[lane].rbegin(); it != lists[lane].rend(); ++it)
                    if ((*it)->segIndex == i && (*it)->dis >= dis) return *it;
            return nullptr;
        }
        for (size_t i = segIndex; i < segVeh[lane].size(); ++i)
            for (auto it = segVeh[lane][i].rbegin(); it != segVeh[lane][i].rend(); ++it)
                if ((*it)->dis >= dis) return *it;
        return nullptr;
    }
    // SimpleLaneChange::estimateGap lanechange.cpp:220-225
    double estimateGap(const Veh &v, int lane) const {
        Veh *leader = vehicleAfter(lane, v.dis, v.segIndex);
        if (!leader) return net.laneLength[lane] - v.dis;
        return leader->dis - v.dis - leader->t.len;
    }
    // LaneChange::getDirection lanechange.cpp:104-113
    int lcDirection(const Veh &v) const {
        if (isLink(v.drivable)) return 0;
        if (!v.sigSend) return 0;
        if (v.sigSend->target < 0) return 0;
        if (v.sigSend->target == outerLane(v.drivable)) return 1;
        if (v.sigSend->target == innerLane(v.drivable)) return -1;
        return 0;
    }
    // SimpleLaneChange::makeSignal lanechange.cpp:152-187 (+ LaneChange::makeSignal lanechange.h:73)
    void makeSignal(Veh &v) {
        if (v.changing) return;
        if (currentTime() - v.lastChangeTime < 3) return;   // coolingTime, lanechange.h:46
        v.sigSend = std::make_shared<Veh::Signal>();
        v.sigSend->source = &v;
        if (!isLink(v.drivable)) {
            const int cur = v.drivable;
            if (net.laneLength[cur] - v.dis < 30) return;
            double curEst = v.gap;
            double outerEst = 0;
            double expectedGap = 2 * v.t.len + 4 * interval * v.t.maxSpeed;
            if (v.gap > expectedGap || v.gap < 1.5 * v.t.len) return;
            if (net.laneIdx[cur] < net.roadNumLanes(net.laneRoad[cur]) - 1) {
                if (onLastRoad(v) || routerNextOf(v, outerLane(cur)) >= 0) {
                    outerEst = estimateGap(v, outerLane(cur));
                    if (outerEst > curEst + v.t.len) v.sigSend->target = outerLane(cur);
                }
            }
            if (net.laneIdx[cur] > 0) {
                if (onLastRoad(v) || routerNextOf(v, innerLane(cur)) >= 0) {
                    double innerEst = estimateGap(v, innerLane(cur));
                    if (innerEst > curEst + v.t.len && innerEst > outerEst) v.sigSend->target = innerLane(cur);
                }
            }
            v.sigSend->urgency = 1;
        }
        if (v.sigSend) v.sigSend->direction = lcDirection(v);
    }
    // LaneChange::updateLeaderAndFollower lanechange.cpp:27-62
    void updateLeaderAndFollower(Veh &v) {
        v.targetLeader = v.targetFollower = nullptr;
        const int target = v.sigSend->target;
        v.targetLeader = vehicleAfter(target, v.dis, v.segIndex);
        const int cur = v.drivable;
        v.leaderGap = v.followerGap = std::numeric_limits<double>::max();
        if (!v.targetLeader) {
            double rest = net.laneLength[cur] - v.dis;
            v.leaderGap = rest;
            double gap = std::numeric_limits<double>::max();
            for (int ll : net.laneOutLinks[target]) {
                Veh *leader = lastVeh(nLanes() + ll);
                if (leader && leader->dis + rest < gap) {
                    gap = leader->dis + rest;
                    if (gap < leader->t.len) {
                        v.targetLeader = leader;
                        v.leaderGap = rest - (leader->t.len - gap);
                    }
                }
            }
        } else {
            v.leaderGap = v.targetLeader->dis - v.dis - v.targetLeader->t.len;
        }
        v.targetFollower = vehicleBefore(target, v.dis, v.segIndex);
        if (v.targetFollower) v.followerGap = v.dis - v.targetFollower->dis - v.t.len;
        else v.followerGap = std::numeric_limits<double>::max();
    }
    // Vehicle::receiveSignal vehicle.cpp:391-402
    static void receiveSignal(Veh &me, Veh &sender) {
        if (me.changing) return;
        int curPriority = me.sigRecv ? me.sigRecv->source->priority : -1;
        int newPriority = sender.priority;
        if ((!me.sigRecv || curPriority < newPriority) && (!me.sigSend || me.priority < newPriority))
            me.sigRecv = sender.sigSend;
    }
    // LaneChange::clearSignal lanechange.cpp:129-139
    static void clearSignal(Veh &v) {
        v.targetLeader = nullptr;
        v.targetFollower = nullptr;
        v.lastDir = v.sigSend ? v.sigSend->direction : 0;
        if (v.changing) return;
        v.sigSend = nullptr;
        v.sigRecv = nullptr;
    }
    double safeGapBefore(const Veh &v) const { return v.targetFollower ? minBrakeDistance(*v.targetFollower) : 0; }  // lanechange.cpp:212-214
    // SimpleLaneChange::yieldSpeed lanechange.cpp:189-210
    double yieldSpeed(Veh &v) {
        if (v.planChange()) v.waitingTime += interval;
        if (v.sigRecv) {
            Veh *source = v.sigRecv->source;
            if (&v == source->targetLeader) return 100;
            double srcSpeed = source->t.speed;
            double gap = source->followerGap - safeGapBefore(*source);
            double s = noCollisionSpeed(srcSpeed, source->t.maxNegAcc, v.t.speed, v.t.maxNegAcc, gap, interval, 0);
            if (s < 0) s = 100;
            return s;
        }
        return 100;
    }
    // Engine::insertShadow engine.cpp:811-819, Vehicle copy ctor vehicle.cpp:27-36,
    // LaneChange::insertShadow lanechange.cpp:73-102
    void insertShadow(Veh &v) {
        Veh *sh = new Veh();
        sh->t = v.t;
        // ControllerInfo copy (vehicle.cpp:15-17); Router copy restarts its road cursor and forgets the
        // planned drivables (router.cpp:11-14)
        sh->dis = v.dis; sh->drivable = v.drivable; sh->prevDrivable = v.prevDrivable;
        sh->approachDist = v.approachDist; sh->gap = v.gap; sh->enterLaneLinkTime = v.enterLaneLinkTime;
        sh->leader = v.leader; sh->blocker = v.blocker; sh->running = v.running;
        sh->route = v.route; sh->iCur = 0; sh->routeValid = false;
        // LaneChangeInfo and Buffer are copied member-wise
        sh->partnerType = v.partnerType; sh->partner = v.partner; sh->offset = v.offset; sh->segIndex = v.segIndex;
        sh->bDisSet = v.bDisSet; sh->bSpeedSet = v.bSpeedSet; sh->bDrvSet = v.bDrvSet; sh->bEndSet = v.bEndSet;
        sh->bBlockerSet = v.bBlockerSet; sh->bEnterSet = v.bEnterSet; sh->bCustomSet = v.bCustomSet;
        sh->bDis = v.bDis; sh->bDelta = v.bDelta; sh->bSpeed = v.bSpeed; sh->bCustom = v.bCustom;
        sh->bDrv = v.bDrv; sh->bEnd = v.bEnd; sh->bBlocker = v.bBlocker; sh->bEnter = v.bEnter;
        sh->flow = v.flow; sh->cnt = v.cnt;   // id + "_shadow": same (flow, cnt), told apart by priority
        sh->enterTime = v.enterTime;
        if (deferShadowPriority) sh->priority = INT_MIN;   // device form: drawn after all roads are done
        else {
            do { sh->priority = (int) rnd(); } while (pool.count(sh->priority));
            pool.emplace(sh->priority, sh);
            shadowsThisStep.emplace_back(&v, sh->priority);
        }
        // LaneChange::insertShadow
        v.changing = true;
        v.waitingTime = 0;
        const int target = v.sigSend->target;
        sh->partnerType = 2; sh->partner = &v;     // setParent
        v.partnerType = 1; v.partner = sh;         // setShadow
        sh->blocker = nullptr;
        sh->drivable = target;
        routerUpdate(*sh);
        auto &L = lists[target];
        auto pos = L.end();
        if (v.targetFollower) {  // targetFollower->getListIterator(): looked up through ITS segment (vehicle.cpp:404-411)
            if (deviceForm) pos = std::find(L.begin(), L.end(), v.targetFollower);
            else {
                auto &sv = segVeh[target][v.targetFollower->segIndex];
                if (std::find(sv.begin(), sv.end(), v.targetFollower) != sv.end())
                    pos = std::find(L.begin(), L.end(), v.targetFollower);
            }
        }
        L.insert(pos, sh);
        if (!deviceForm) {   // Segment::insertVehicle roadnet.cpp:944-948 (into the segment with the PARENT's index)
            auto &sv = segVeh[target][v.segIndex];
            auto it = sv.begin();
            for (; it != sv.end() && (*it)->dis > sh->dis; ++it) {}
            sv.insert(it, sh);
            // the planned device form reads a segment as "the list filtered by segmentIndex": count
            // the cases where the segment list is NOT that subsequence (needs two equal distances)
            std::vector<Veh *> sub;
            for (Veh *x : L) if (x->segIndex == v.segIndex) sub.push_back(x);
            if (sub != sv) ++segOrderMismatch;
        }
        updateLeaderAndGap(*sh, v.targetLeader);
        if (v.targetFollower) updateLeaderAndGap(*v.targetFollower, sh);
        activeCount++;
    }
    // Engine::threadPlanLaneChange engine.cpp:374-389 + Engine::scheduleLaneChange :792-809
    void planLaneChange() {
        std::vector<Veh *> buffer;
        for (auto &kv : pool) {
            Veh *v = kv.second;
            if (v->running && v->isReal()) {
                makeSignal(*v);
                if (v->planChange()) buffer.push_back(v);
            }
        }
        // same library sort and comparator as the reference: with every urgency equal to 1 the
        // (unstable) result is a function of the input order alone
        std::sort(buffer.begin(), buffer.end(), [](Veh *a, Veh *b) { return a->sigSend->urgency > b->sigSend->urgency; });
        if (deviceForm) { scheduleByRoad(buffer); return; }
        for (Veh *v : buffer) {
            updateLeaderAndFollower(*v);
            if (v->targetLeader) receiveSignal(*v->targetLeader, *v);      // SimpleLaneChange::sendSignal lanechange.cpp:207-210
            if (v->targetFollower) receiveSignal(*v->targetFollower, *v);
            if (v->planChange() && (v->sigSend && !v->sigRecv) && !v->changing) {
                const bool gapValid = v->leaderGap >= minBrakeDistance(*v) && v->followerGap >= safeGapBefore(*v);  // lanechange.h:79
                if (gapValid && !isLink(v->drivable)) insertShadow(*v);
            }
        }
    }
    // Device form of scheduleLaneChange: candidates of different roads never interact (a candidate
    // reads its road's lanes and the laneLinks leaving them, writes signals of vehicles on those), so
    // every road walks ITS candidates in the global order, roads in any order (here: descending);
    // the shadows' priorities -- the only global coupling, through the RNG -- are drawn afterwards
    // in the global order.
    void scheduleByRoad(const std::vector<Veh *> &buffer) {
        std::vector<std::vector<Veh *>> byRoad(net.nRoads());
        for (Veh *v : buffer) byRoad[net.laneRoad[v->drivable]].push_back(v);   // candidates are on lanes (planChange)
        statCandidates += (long long) buffer.size();
        statMaxCandidates = std::max(statMaxCandidates, (int) buffer.size());
        for (auto &b : byRoad) statMaxCandidatesPerRoad = std::max(statMaxCandidatesPerRoad, (int) b.size());
        deferShadowPriority = true;
        for (int r = net.nRoads() - 1; r >= 0; --r)
            for (Veh *v : byRoad[r]) {
                updateLeaderAndFollower(*v);
                if (v->targetLeader) receiveSignal(*v->targetLeader, *v);
                if (v->targetFollower) receiveSignal(*v->targetFollower, *v);
                if (v->planChange() && (v->sigSend && !v->sigRecv) && !v->changing) {
                    const bool gapValid = v->leaderGap >= minBrakeDistance(*v) && v->followerGap >= safeGapBefore(*v);
                    if (gapValid && !isLink(v->drivable)) insertShadow(*v);
                }
            }
        deferShadowPriority = false;
        for (Veh *v : buffer)
            if (v->partnerType == 1 && v->partner->priority == INT_MIN) {   // got its shadow in this step
                Veh *sh = v->partner;
                do { sh->priority = (int) rnd(); } while (pool.count(sh->priority));
                pool.emplace(sh->priority, sh);
            }
    }
    bool deferShadowPriority = false;
    void (*lcProbe)(Oracle &, int) = nullptr;
    // for tests/device_step_probe.cpp (the device code emulated on the host): this step's spawns in
    // planRoute order and this step's shadows (parent, priority drawn) in creation order
    std::vector<Veh *> spawnedThisStep;
    std::vector<std::pair<Veh *, int>> shadowsThisStep;
    long long segOrderMismatch = 0;
    // sizes of the sequential parts of the device form, summed / maximised over the steps so far
    long long statCandidates = 0, statInvolved = 0, statRunning = 0;
    int statMaxCandidatesPerRoad = 0, statMaxInvolved = 0, statMaxCandidates = 0;
    // Device form of threadGetAction: pass 1 in arbitrary (here: descending priority) order computes
    // what does not depend on the order; pass 2 finishes the plain vehicles in arbitrary order and
    // only the vehicles involved in a lane change (a partner, or a received signal) in ascending
    // priority, as the reference's single worker does.
    void controlDeviceForm() {
        for (auto it = pool.rbegin(); it != pool.rend(); ++it)
            if (it->second->running) it->second->ctlHead = nextSpeedHead(*it->second);
        if (lcProbe) lcProbe(*this, 2);        // tests/lc_device_probe.cpp: heads computed, nothing finished yet
        std::vector<Veh *> involved;
        for (auto it = pool.rbegin(); it != pool.rend(); ++it) {
            Veh *v = it->second;
            if (!v->running) continue;
            if (v->partner || v->sigRecv || v->partnerType != 0 || v->changing) involved.push_back(v);
            else vehicleControl(*v);
        }
        statInvolved += (long long) involved.size();
        statMaxInvolved = std::max(statMaxInvolved, (int) involved.size());
        statRunning += (long long) activeCount;
        for (auto it = involved.rbegin(); it != involved.rend(); ++it) vehicleControl(**it);   // ascending priority
        if (lcProbe) lcProbe(*this, 3);
    }
    // LaneChange::finishChanging lanechange.cpp:115-127 + Vehicle::finishChanging vehicle.cpp:378-381
    void finishChanging(Veh &v) {
        v.changing = false;
        v.lcFinished = true;
        v.lastChangeTime = currentTime();
        Veh *partner = v.partner;
        partner->partnerType = 0;     // (and takes over the name: same (flow, cnt) here)
        partner->offset = 0;
        partner->partner = nullptr;
        v.partner = nullptr;
        clearSignal(v);
        v.bEnd = true; v.bEndSet = true;
    }
    // Vehicle::abortLaneChange vehicle.cpp:413-417 + LaneChange::abortChanging lanechange.cpp:141-148
    void abortLaneChange(Veh &v) {
        v.bEnd = true; v.bEndSet = true;
        Veh *partner = v.partner;
        partner->changing = false;
        partner->partnerType = 0;
        partner->offset = 0;
        partner->partner = nullptr;
        clearSignal(v);
    }
    // vehicle.cpp:49-68
    void setDeltaDistance(Veh &v, double dis) {
        if (!v.bDisSet || dis < v.bDelta) {
            v.bEndSet = false;
            v.bDrvSet = false;
            v.bDelta = dis;
            dis = dis + v.dis;
            int d = v.drivable;
            for (int i = 0; d >= 0 && dis > drvLength(d); ++i) {
                dis -= drvLength(d);
                int nd = nextDrivable(v, i);
                if (nd < 0) { v.bEnd = true; v.bEndSet = true; }
                d = nd;
                v.bDrv = d;
                v.bDrvSet = true;
            }
            v.bDis = dis;
            v.bDisSet = true;
        }
    }
    // engine.cpp:188-251 (laneChange off)
    void vehicleControl(Veh &v) {
        double ns = v.bSpeedSet ? v.bSpeed : nextSpeed(v);
        if (laneChange) {  // engine.cpp:195-205: a vehicle and its shadow move as one
            Veh *partner = v.partner;
            if (partner != nullptr && !partner->bSpeedSet) {
                double partnerSpeed = nextSpeed(*partner);
                ns = min2(ns, partnerSpeed);
                partner->bSpeed = ns;
                partner->bSpeedSet = true;
                if (partner->bEndSet) { v.bEnd = true; v.bEndSet = true; }
            }
        }
        double deltaDis, speed = v.t.speed;
        if (ns < 0) {
            deltaDis = 0.5 * speed * speed / v.t.maxNegAcc;
            ns = 0;
        } else {
            deltaDis = (speed + ns) * interval / 2;
        }
        v.bSpeed = ns;
        v.bSpeedSet = true;
        setDeltaDistance(v, deltaDis);
        if (laneChange) {  // engine.cpp:224-244
            if (!v.isReal() && v.bDrvSet && v.bDrv >= 0) abortLaneChange(v);   // getChangedDrivable() != nullptr
            if (v.changing) {
                int dir = v.sigSend ? v.sigSend->direction : 0;
                const double curWidth = isLink(v.drivable) ? 0.0 : net.laneWidth[v.drivable];   // (getCurLane() on a laneLink is undefined in the reference)
                const double maxOffset = (net.laneWidth[v.sigSend->target] + curWidth) / 2;   // vehicle.h:347-350
                double newOffset = std::fabs(v.offset + max2(0.2 * ns, 1) * interval * dir);
                newOffset = min2(newOffset, maxOffset);
                v.offset = newOffset * dir;
                if (newOffset >= maxOffset) finishChanging(v);
            }
        }
        if (!v.bEndSet && v.bDrvSet) pushBuffer.emplace_back(&v, v.bDis);
    }
    // vehicle.cpp:107-143
    void commit(Veh &v) {
        if (v.bEndSet) v.bEndSet = false;
        if (v.bDisSet) { v.dis = v.bDis; v.bDisSet = false; }
        if (v.bSpeedSet) { v.t.speed = v.bSpeed; v.bSpeedSet = false; }
        if (v.bCustomSet) v.bCustomSet = false;
        if (v.bDrvSet) {
            v.prevDrivable = v.drivable;
            v.drivable = v.bDrv;
            v.bDrvSet = false;
            routerUpdate(v);
        }
        if (v.bEnterSet) { v.enterLaneLinkTime = v.bEnter; v.bEnterSet = false; }
        if (v.bBlockerSet) { v.blocker = v.bBlocker; v.bBlockerSet = false; }
        else v.blocker = nullptr;
    }
    // vehicle.cpp:157-196
    void updateLeaderAndGap(Veh &v, Veh *leader) {
        if (leader != nullptr && leader->drivable == v.drivable) {
            v.leader = leader;
            v.gap = leader->dis - leader->t.len - v.dis;
            return;
        }
        v.leader = nullptr;
        double dis = drvLength(v.drivable) - v.dis;
        for (int i = 0;; ++i) {
            int d = nextDrivable(v, i);
            if (d < 0) return;
            if (isLink(d)) {
                int startLane = net.llStartLane[d - nLanes()];
                for (int ll : net.laneOutLinks[startLane]) {
                    Veh *cand = lastVeh(nLanes() + ll);
                    if (cand != nullptr) {
                        double candGap = dis + cand->dis - cand->t.len;
                        if (v.leader == nullptr || candGap < v.gap) {
                            v.leader = cand;
                            v.gap = candGap;
                        }
                    }
                }
                if (v.leader) return;
            } else {
                if ((v.leader = lastVeh(d)) != nullptr) {
                    v.gap = dis + v.leader->dis - v.leader->t.len;
                    return;
                }
            }
            dis += drvLength(d);
            if (dis > v.t.maxSpeed * v.t.maxSpeed / v.t.usualNegAcc / 2 + v.t.maxSpeed * interval * 2) return;
        }
    }

    // ---------------- Engine phases ----------------
    // Vehicle ctor vehicle.cpp:38-47 + Engine::pushVehicle engine.cpp:605-613
    Veh *newVehicle(const VehicleTemplate &t, const std::vector<int> &anchors, int flow, int cnt) {
        Veh *v = new Veh();
        v->t = t;
        v->flow = flow;
        v->cnt = cnt;
        v->route = anchors;  // anchor points until updateShortestPath
        v->approachDist = t.maxSpeed * t.maxSpeed / t.usualNegAcc / 2 + t.maxSpeed * interval * 2;
        do { v->priority = (int) rnd(); } while (pool.count(v->priority));
        v->enterTime = currentTime();
        (void) rnd();  // threadIndex = rnd() % threadNum, drawn even with one thread
        pool.emplace(v->priority, v);
        return v;
    }
    // flow.cpp:6-22
    void flowStep(FlowState &f, int index) {
        if (!f.valid) return;
        if (f.def.endTime != -1 && f.currentTime > f.def.endTime) return;
        if (f.currentTime >= f.def.startTime) {
            while (f.nowTime >= f.def.interval) {
                Veh *v = newVehicle(f.def.tmpl, f.def.anchors, index, f.cnt++);
                planRouteBuffer[f.def.anchors[0]].push_back(v);
                f.nowTime -= f.def.interval;
            }
            f.nowTime += interval;
        }
        f.currentTime += interval;
    }
    // engine.cpp:450-470 (+ threadPlanRoute :272-280, Router::getFirstDrivable router.cpp:23-37)
    void planRoute() {
        for (int r = 0; r < net.nRoads(); ++r) {
            for (Veh *v : planRouteBuffer[r]) {
                std::vector<int> roads;
                v->routeValid = routing->resolve(v->route, roads);
                if (v->routeValid) {
                    v->route = roads;
                    v->iCur = 0;
                    v->planned.clear();
                    std::vector<int> cand;
                    for (int l = net.roadLaneBeg[roads[0]]; l < net.roadLaneBeg[roads[0] + 1]; ++l) {
                        std::vector<int> tmp;
                        net.linksToRoad(l, roads[1], tmp);
                        if (!tmp.empty()) cand.push_back(l);
                    }
                    v->drivable = cand[rnd() % cand.size()];
                    waiting[v->drivable].push_back(v);
                    v->firstLaneForProbe = v->drivable;
                    v->initialSpeedForProbe = v->t.speed;
                    spawnedThisStep.push_back(v);
                } else {
                    if (v->flow >= 0) {
                        if (flows[v->flow].valid)
                            std::cerr << "[warning] Invalid route '" << flows[v->flow].def.id << "'. Omitted by default." << std::endl;
                        flows[v->flow].valid = false;
                    }
                    pool.erase(v->priority);
                    delete v;
                }
            }
            planRouteBuffer[r].clear();
        }
    }
    // engine.cpp:502-516, Lane::available roadnet.cpp:428-435
    void handleWaiting() {
        for (int l = 0; l < nLanes(); ++l) {
            auto &buf = waiting[l];
            if (buf.empty()) continue;
            Veh *v = buf.front();
            Veh *tail = lastVeh(l);
            bool available = !tail || tail->dis > tail->t.len + v->t.minGap;
            if (available) {
                v->running = true;
                activeCount += 1;
                lists[l].push_back(v);
                updateLeaderAndGap(*v, tail);
                buf.pop_front();
            }
        }
    }
    // engine.cpp:317-372
    void notifyCross() {
        for (int s = 0; s < 2; ++s) std::fill(notifyVeh[s].begin(), notifyVeh[s].end(), nullptr);
        for (int ll = 0; ll < net.nLinks(); ++ll) {
            const auto &crosses = net.llCrosses[ll];
            int ri = (int) crosses.size() - 1;  // reverse iterator
            auto dist = [&](int k) { return net.crossDist[crosses[k].side][crosses[k].cross]; };
            auto notify = [&](int k, Veh *v, double d) {
                notifyVeh[crosses[k].side][crosses[k].cross] = v;
                notifyDist[crosses[k].side][crosses[k].cross] = d;
            };
            const int linkDrv = nLanes() + ll;
            Veh *v = lastVeh(net.llEndLane[ll]);
            if (v && v->prevDrivable == linkDrv) {
                double vehDistance = v->dis - v->t.len;
                while (ri >= 0) {
                    double crossDistance = net.llLength[ll] - dist(ri);
                    if (crossDistance + vehDistance < 0) {  // leaveDistance = 0, roadnet.h:126
                        notify(ri, v, -(v->dis + crossDistance));
                        --ri;
                    } else break;
                }
            }
            for (Veh *lv : lists[linkDrv]) {
                double vehDistance = lv->dis;
                while (ri >= 0) {
                    double crossDistance = dist(ri);
                    if (vehDistance > crossDistance) {
                        if (vehDistance - crossDistance - lv->t.len <= 0) notify(ri, lv, crossDistance - vehDistance);
                        else break;
                    } else {
                        notify(ri, lv, crossDistance - vehDistance);
                    }
                    --ri;
                }
            }
            v = firstVeh(net.llStartLane[ll]);
            if (v && nextDrivable(*v) == linkDrv && linkAvailable(ll)) {
                double vehDistance = net.laneLength[net.llStartLane[ll]] - v->dis;
                while (ri >= 0) {
                    notify(ri, v, vehDistance + dist(ri));
                    --ri;
                }
            }
        }
    }
    // engine.cpp:282-315 + :477-494
    void updateLocation() {
        for (size_t d = 0; d < lists.size(); ++d) {
            auto &L = lists[d];
            size_t w = 0;
            for (size_t k = 0; k < L.size(); ++k) {
                Veh *v = L[k];
                bool changed = v->bDrvSet;  // getChangedDrivable() != nullptr  (null target handled by bEndSet)
                if (!(changed && v->bDrv >= 0) && !v->bEndSet) L[w++] = v;
                if (v->bEndSet) {
                    removeBuffer.insert(v);
                    if (!v->lcFinished) {  // engine.cpp:297-301: a vehicle replaced by its shadow is not "finished"
                        finishedCnt += 1;
                        cumulativeTravelTime += currentTime() - v->enterTime;
                    }
                    pool.erase(v->priority);
                    activeCount--;
                }
            }
            L.resize(w);
        }
        // tie order inside std::sort is unspecified in the reference; here: stable, pool order
        for (size_t a = 0; a + 1 < pushBuffer.size(); ++a)
            for (size_t b = a + 1; b < pushBuffer.size(); ++b)
                if (pushBuffer[a].second == pushBuffer[b].second && pushBuffer[a].first->bDrv == pushBuffer[b].first->bDrv) {
                    ++ties;
                    if (getenv("CFO_PRINT_TIES"))
                        fprintf(stderr, "[oracle] tie at step %zu: drivable %d dis %.17g  flow_%d_%d (from %d, speed %.17g) vs flow_%d_%d (from %d, speed %.17g)\n", step,
                                pushBuffer[a].first->bDrv, pushBuffer[a].second, pushBuffer[a].first->flow, pushBuffer[a].first->cnt, pushBuffer[a].first->drivable, pushBuffer[a].first->bSpeed,
                                pushBuffer[b].first->flow, pushBuffer[b].first->cnt, pushBuffer[b].first->drivable, pushBuffer[b].first->bSpeed);
                }
        std::stable_sort(pushBuffer.begin(), pushBuffer.end(),
                         [](const std::pair<Veh *, double> &a, const std::pair<Veh *, double> &b) { return a.second > b.second; });
        for (auto &pr : pushBuffer) {
            Veh *v = pr.first;
            if (v->bDrvSet && v->bDrv >= 0) {
                lists[v->bDrv].push_back(v);
                v->bEnter = isLink(v->bDrv) ? (int64_t) step : (int64_t) INT_MAX;
                v->bEnterSet = true;
            }
        }
        pushBuffer.clear();
    }
    // engine.cpp:415-427 + :496-500
    void updateAction() {
        for (auto &kv : pool) {
            Veh *v = kv.second;
            if (!v->running) continue;
            if (removeBuffer.count(v->bBlocker)) {  // setBlocker(nullptr)
                v->bBlocker = nullptr;
                v->bBlockerSet = true;
            }
            commit(*v);
            clearSignal(*v);   // engine.cpp:424 (no-op without lane change: nothing is ever set)
        }
        for (Veh *v : removeBuffer) delete v;
        removeBuffer.clear();
    }
    // engine.cpp:429-442
    void updateLeaderAndGapAll() {
        for (auto &L : lists) {
            Veh *leader = nullptr;
            for (Veh *v : L) {
                updateLeaderAndGap(*v, leader);
                leader = v;
            }
        }
    }
    // trafficlight.cpp:29-37
    void lights() {
        if (rlTrafficLight) return;
        for (int i = 0; i < net.nInter(); ++i) {
            if (net.interVirtual[i]) continue;
            int nph = net.interPhaseBeg[i + 1] - net.interPhaseBeg[i];
            remain[i] -= interval;
            while (remain[i] <= 0.0) {
                curPhase[i] = (curPhase[i] + 1) % nph;
                remain[i] += net.phaseTime[net.interPhaseBeg[i] + curPhase[i]];
            }
        }
    }
    // engine.cpp:566-594
    void nextStep() {
        spawnedThisStep.clear();
        shadowsThisStep.clear();
        for (size_t i = 0; i < flows.size(); ++i) flowStep(flows[i], (int) i);
        planRoute();
        handleWaiting();
        if (laneChange) {  // engine.cpp:570-574
            if (lcProbe) lcProbe(*this, 0);    // tests/lc_device_probe.cpp: state right before the lane-change phases
            initSegments();
            planLaneChange();
            if (lcProbe) lcProbe(*this, 1);    // ... and right after scheduling
            updateLeaderAndGapAll();
        }
        notifyCross();
        // threadGetAction: running vehicles; order only matters for pushBuffer ties
        if (deviceForm) controlDeviceForm();
        else
            for (auto &kv : pool)
                if (kv.second->running) vehicleControl(*kv.second);
        updateLocation();
        updateAction();
        updateLeaderAndGapAll();
        lights();
        step += 1;
    }
    void initLights() {  // TrafficLight::init(0), trafficlight.cpp:6-11
        curPhase.assign(net.nInter(), 0);
        remain.assign(net.nInter(), 0.0);
        for (int i = 0; i < net.nInter(); ++i)
            if (!net.interVirtual[i]) remain[i] = net.phaseTime[net.interPhaseBeg[i]];
    }
    // engine.cpp:744-760
    void reset(bool resetRnd) {
        for (auto &kv : pool) delete kv.second;
        pool.clear();
        for (auto &L : lists) L.clear();
        for (auto &w : waiting) w.clear();
        for (auto &b : planRouteBuffer) b.clear();
        initLights();
        finishedCnt = 0;
        cumulativeTravelTime = 0;
        for (auto &f : flows) {  // flow.cpp:28-32
            f.nowTime = f.def.interval;
            f.currentTime = 0;
            f.cnt = 0;
        }
        step = 0;
        activeCount = 0;
        if (resetRnd) rnd.seed(seed);
    }
    bool load(const std::string &configFile) {  // engine.cpp:37-84
        bool opened = false;
        cfb::Json doc = cfb::Json::parseFile(configFile, &opened);
        if (!opened || !doc.isObject()) return false;
        auto get = [&](const char *k) -> const cfb::Json & {
            const cfb::Json *v = doc.find(k);
            if (!v) throw cfb::JsonError(std::string(k) + " is required but missing in json file");
            return *v;
        };
        interval = get("interval").asDouble();
        rlTrafficLight = get("rlTrafficLight").asBool();
        if (const cfb::Json *lc = doc.find("laneChange")) laneChange = lc->isBool() && lc->asBool();   // engine.cpp:52 (optional, default false)
        seed = get("seed").asInt();
        rnd.seed(seed);
        std::string dir = get("dir").s;
        if (!net.load(dir + get("roadnetFile").s)) return false;
        std::vector<cfb::FlowDef> defs;
        if (!cfb::loadFlows(dir + get("flowFile").s, net, defs)) return false;
        for (auto &d : defs) {
            FlowState f;
            f.def = d;
            f.nowTime = d.interval;  // flow.h:35
            flows.push_back(f);
        }
        routing = new cfb::Routing(net);
        lists.resize(net.nDrivables());
        waiting.resize(net.nLanes());
        planRouteBuffer.resize(net.nRoads());
        for (int s = 0; s < 2; ++s) {
            notifyVeh[s].assign(net.nCross(), nullptr);
            notifyDist[s].assign(net.nCross(), 0.0);
        }
        initLights();
        // Road::buildSegmentationByInterval roadnet.cpp:687-691 with (len + minGap) * MAX_NUM_CARS_ON_SEGMENT
        // of a default VehicleInfo = (5 + 2) * 10 (roadnet.cpp:305-312, config.h:5); Lane::buildSegmentation :852-861
        segStart.resize(net.nLanes());
        segVeh.resize(net.nLanes());
        for (int r = 0; r < net.nRoads(); ++r) {
            double len = 0.0;
            const auto &pts = net.roadPoints[r];
            for (size_t i = 0; i + 1 < pts.size(); ++i) {
                const double dx = pts[i + 1].x - pts[i].x, dy = pts[i + 1].y - pts[i].y;
                len += sqrt(dx * dx + dy * dy);
            }
            const double segInterval = (5.0 + 2.0) * 10;
            const size_t numSegs = std::max((size_t) ceil(len / segInterval), (size_t) 1);
            for (int l = net.roadLaneBeg[r]; l < net.roadLaneBeg[r + 1]; ++l) {
                segStart[l].resize(numSegs);
                segVeh[l].assign(numSegs, {});
                for (size_t i = 0; i < numSegs; ++i) segStart[l][i] = i * net.laneLength[l] / numSegs;
            }
        }
        return true;
    }
    ~Oracle() {
        for (auto &kv : pool) delete kv.second;
        delete routing;
    }
};

}  // namespace

// ------------------------------------------------------------------------------------------
// Plain C interface for ctypes (tests, smoke, bench cpu_baseline).
extern "C" {

struct OracleVehRec {   // mirrors the per-vehicle record of `refdump run`
    int32_t flow, cnt, priority, drivable, leaderFlow, leaderCnt, blockerFlow, blockerCnt;
    double dis, speed, gap;
    int64_t enterLaneLinkTime;
};

void *cfo_create(const char *config) {
    Oracle *o = new Oracle();
    try {
        if (!o->load(config)) { delete o; return nullptr; }
    } catch (const std::exception &e) {
        std::cerr << e.what() << std::endl;
        delete o;
        return nullptr;
    }
    return o;
}
void cfo_destroy(void *h) { delete (Oracle *) h; }
void cfo_next_step(void *h, int n) { for (int i = 0; i < n; ++i) ((Oracle *) h)->nextStep(); }
void cfo_reset(void *h, int reseed) { ((Oracle *) h)->reset(reseed != 0); }
int cfo_num_lanes(void *h) { return ((Oracle *) h)->net.nLanes(); }
int cfo_num_drivables(void *h) { return ((Oracle *) h)->net.nDrivables(); }
int cfo_num_intersections(void *h) { return ((Oracle *) h)->net.nInter(); }
int cfo_vehicle_count(void *h) { return (int) ((Oracle *) h)->activeCount; }
int cfo_pool_size(void *h) { return (int) ((Oracle *) h)->pool.size(); }
int cfo_finished_count(void *h) { return ((Oracle *) h)->finishedCnt; }
double cfo_cumulative_travel_time(void *h) { return ((Oracle *) h)->cumulativeTravelTime; }
int cfo_tie_count(void *h) { return ((Oracle *) h)->ties; }
int cfo_max_refused_cross_index(void *h) { return ((Oracle *) h)->maxRefusedCross; }
double cfo_current_time(void *h) { return ((Oracle *) h)->currentTime(); }
void cfo_lane_vehicle_count(void *h, int32_t *out) {  // engine.cpp:628-634
    Oracle *o = (Oracle *) h;
    for (int l = 0; l < o->nLanes(); ++l) out[l] = (int32_t) o->lists[l].size();
}
void cfo_lane_waiting_count(void *h, int32_t *out) {  // engine.cpp:636-648
    Oracle *o = (Oracle *) h;
    for (int l = 0; l < o->nLanes(); ++l) {
        int c = 0;
        for (Veh *v : o->lists[l]) c += v->t.speed < 0.1;
        out[l] = c;
    }
}
void cfo_lane_queue_size(void *h, int32_t *out) {
    Oracle *o = (Oracle *) h;
    for (int l = 0; l < o->nLanes(); ++l) out[l] = (int32_t) o->waiting[l].size();
}
void cfo_phases(void *h, int32_t *out) {
    Oracle *o = (Oracle *) h;
    for (int i = 0; i < o->net.nInter(); ++i) out[i] = o->net.interVirtual[i] ? -1 : o->curPhase[i];
}
void cfo_set_tl_phase(void *h, int inter, int phase) {  // engine.cpp:719-725
    Oracle *o = (Oracle *) h;
    if (!o->rlTrafficLight) return;
    o->curPhase[inter] = phase;
}
// Engine::pushVehicle(info, roads) engine.cpp:693-717 (values: NaN = keep the struct default)
void cfo_push_vehicle(void *h, const double *v, const int32_t *roads, int n) {
    Oracle *o = (Oracle *) h;
    VehicleTemplate t;
    double *f[10] = {&t.speed, &t.len, &t.width, &t.maxPosAcc, &t.maxNegAcc, &t.usualPosAcc, &t.usualNegAcc,
                     &t.minGap, &t.maxSpeed, &t.headwayTime};
    for (int k = 0; k < 10; ++k) if (v[k] == v[k]) *f[k] = v[k];
    std::vector<int> anchors(roads, roads + n);
    Veh *veh = o->newVehicle(t, anchors, -2, o->manuallyPushCnt++);
    o->planRouteBuffer[anchors[0]].push_back(veh);
}
// Engine::setVehicleSpeed engine.cpp:827-834 -> Vehicle::setCustomSpeed vehicle.h:128-131; -1 = no such vehicle
int cfo_set_vehicle_speed(void *h, int flow, int cnt, double speed) {
    Oracle *o = (Oracle *) h;
    for (auto &kv : o->pool) {
        Veh *v = kv.second;
        if (v->flow == flow && v->cnt == cnt && v->isReal()) {
            v->bCustom = speed;
            v->bCustomSet = true;
            return 0;
        }
    }
    return -1;
}
// Engine::setRoute engine.cpp:852-866 -> Router::setRoute router.cpp:245-264: 1 = the vehicle now follows
// [current road] + roads, 0 = refused (on a laneLink, unreachable, or the current lane cannot continue), -1 = no such vehicle
int cfo_set_vehicle_route(void *h, int flow, int cnt, const int32_t *roads, int n) {
    Oracle *o = (Oracle *) h;
    for (auto &kv : o->pool) {
        Veh *v = kv.second;
        if (!(v->flow == flow && v->cnt == cnt && v->isReal())) continue;
        if (v->drivable < 0 || o->isLink(v->drivable)) return 0;
        const int curRoad = v->route[v->iCur];
        std::vector<int> anchors{curRoad};
        anchors.insert(anchors.end(), roads, roads + n);
        std::vector<int> backup = v->route, fresh;
        const int backupCur = v->iCur;
        bool ok = o->routing->resolve(anchors, fresh);   // Router::updateShortestPath router.cpp:228-243
        v->planned.clear();
        if (ok) { v->route = fresh; v->iCur = 0; }
        if (ok && o->onValidLane(*v)) return 1;
        v->route = backup;
        v->planned.clear();
        v->iCur = backupCur;   // the road cursor goes back to cur_road (router.cpp:258-260)
        return 0;
    }
    return -1;
}
// Engine::getLeader engine.cpp:836-850: 1 + (flow, cnt) of the leader, 0 = none, -1 = no such vehicle
int cfo_get_leader(void *h, int flow, int cnt, int32_t *leaderFlow, int32_t *leaderCnt) {
    Oracle *o = (Oracle *) h;
    for (auto &kv : o->pool) {
        Veh *v = kv.second;
        if (v->flow == flow && v->cnt == cnt && v->isReal()) {
            if (!v->leader) return 0;
            *leaderFlow = v->leader->flow; *leaderCnt = v->leader->cnt;
            return 1;
        }
    }
    return -1;
}
void cfo_set_random_seed(void *h, int seed) { ((Oracle *) h)->rnd.seed(seed); }  // Engine::setRandomSeed engine.h:170
int cfo_road_index(void *h, const char *id) {
    Oracle *o = (Oracle *) h;
    auto it = o->net.roadIndex.find(id);
    return it == o->net.roadIndex.end() ? -1 : it->second;
}
// Engine::getAverageTravelTime engine.cpp:682-691
double cfo_average_travel_time(void *h) {
    Oracle *o = (Oracle *) h;
    double tt = o->cumulativeTravelTime;
    int n = o->finishedCnt;
    for (auto &kv : o->pool) { tt += o->currentTime() - kv.second->enterTime; n++; }
    return n == 0 ? 0 : tt / n;
}
// running vehicles in vehiclePool (priority) order, like Engine::getRunningVehicles engine.cpp:780-790
int cfo_vehicles(void *h, OracleVehRec *out, int cap) {
    Oracle *o = (Oracle *) h;
    int n = 0;
    for (auto &kv : o->pool) {
        Veh *v = kv.second;
        if (!v->running) continue;
        if (n < cap) {
            OracleVehRec &r = out[n];
            r.flow = v->flow; r.cnt = v->cnt; r.priority = v->priority; r.drivable = v->drivable;
            r.leaderFlow = v->leader ? v->leader->flow : -1;
            r.leaderCnt = v->leader ? v->leader->cnt : -1;
            r.blockerFlow = v->blocker ? v->blocker->flow : -1;
            r.blockerCnt = v->blocker ? v->blocker->cnt : -1;
            r.dis = v->dis; r.speed = v->t.speed; r.gap = v->leader ? v->gap : 0.0;
            r.enterLaneLinkTime = v->enterLaneLinkTime;
        }
        ++n;
    }
    return n;
}
// laneChange runs: every running vehicle including shadows, vehiclePool order; mirrors `refdump runlc`
struct OracleLcRec {
    int32_t flow, cnt, priority, partnerType, partnerPriority, drivable, leaderPriority, blockerPriority, flags, lastDir;
    double dis, speed, gap, offset, waitingTime, lastChangeTime;
};
int cfo_lc_vehicles(void *h, OracleLcRec *out, int cap) {
    Oracle *o = (Oracle *) h;
    int n = 0;
    for (auto &kv : o->pool) {
        Veh *v = kv.second;
        if (!v->running) continue;
        if (n < cap) {
            OracleLcRec &r = out[n];
            r.flow = v->flow; r.cnt = v->cnt; r.priority = v->priority;
            r.partnerType = v->partnerType;
            r.partnerPriority = v->partner ? v->partner->priority : -1;
            r.drivable = v->drivable;
            r.leaderPriority = v->leader ? v->leader->priority : -1;
            r.blockerPriority = v->blocker ? v->blocker->priority : -1;
            r.flags = (int32_t) v->changing | ((int32_t) v->lcFinished << 1);
            r.lastDir = v->lastDir;
            r.dis = v->dis; r.speed = v->t.speed; r.gap = v->leader ? v->gap : 0.0;
            r.offset = v->offset; r.waitingTime = v->waitingTime; r.lastChangeTime = v->lastChangeTime;
        }
        ++n;
    }
    return n;
}
// list order of one drivable as priorities; returns the count
int cfo_drivable_priorities(void *h, int drivable, int32_t *out, int cap) {
    Oracle *o = (Oracle *) h;
    int n = 0;
    for (Veh *v : o->lists[drivable]) {
        if (n < cap) out[n] = v->priority;
        ++n;
    }
    return n;
}
// running vehicles whose lane cannot continue their route (Router::onValidLane false): the case the GPU
// engine does not handle like the reference yet (DESIGN.md section 6, "Fuzzing")
int cfo_invalid_lane_vehicles(void *h) {
    Oracle *o = (Oracle *) h;
    int n = 0;
    for (auto &kv : o->pool)
        if (kv.second->running && !o->onValidLane(*kv.second)) ++n;
    return n;
}
int cfo_lane_change(void *h) { return ((Oracle *) h)->laneChange ? 1 : 0; }
// switch to the decomposition planned for the GPU (must not change any result; DESIGN.md section 10)
void cfo_device_form_stats(void *h, double out[6]) {
    Oracle *o = (Oracle *) h;
    out[0] = (double) o->statCandidates; out[1] = o->statMaxCandidates; out[2] = o->statMaxCandidatesPerRoad;
    out[3] = (double) o->statInvolved; out[4] = o->statMaxInvolved; out[5] = (double) o->statRunning;
}
// reference-ordered mode: shadow insertions after which a segment list was not the lane list filtered by segment index
long long cfo_segment_order_mismatches(void *h) { return ((Oracle *) h)->segOrderMismatch; }
void cfo_set_device_form(void *h, int on) { ((Oracle *) h)->deviceForm = on != 0; }
// list order of one drivable as (flow,cnt) pairs; returns the count
int cfo_drivable_vehicles(void *h, int drivable, int32_t *out, int cap) {
    Oracle *o = (Oracle *) h;
    int n = 0;
    for (Veh *v : o->lists[drivable]) {
        if (n < cap) { out[2 * n] = v->flow; out[2 * n + 1] = v->cnt; }
        ++n;
    }
    return n;
}

}  // extern "C"
