// device_view.cuh -- device-side data layout (View) and the scalar helpers of the step kernels.
// Part of device_sim.cu (included there, inside namespace cfb's translation unit); a header only so that
// tests/lc_device_probe.cpp can compile the device functions for the host.
#pragma once

namespace cfb {

// ------------------------------------------------------------------------------------------
// Device-side tables
struct DTmpl {  // 16 doubles
    double len, maxPosAcc, maxNegAcc, usualPosAcc, usualNegAcc, minGap, maxSpeed, headwayTime;
    double yieldDistance, turnSpeed, approachDist, speed0, pad[4];
};

struct __align__(16) Notify {  // one side of one Cross (roadnet.h:122-124), epoch-stamped
    double dist;
    int pos;
    int epoch;
    // The terms of Cross::canPass (roadnet.cpp:603-676) that depend on the NOTIFIED vehicle alone -- it is the foe of
    // everybody asking from the crossing link -- evaluated once here by k_notify (one lane per cross, no divergence)
    // instead of once per asking vehicle at the end of k_control's dependent-load chain: see foeTerms().
    int slot, prio, enterLL, steps;   // foe vehicle handle, Vehicle::priority, enterLaneLinkTime, reach steps (dist > 0)
    int flags;                        // NF_* | RoadLinkType of the foe's link << 8
    int pad0, pad1, pad2;
};
constexpr int NF_CAN_YIELD = 1;       // Vehicle::canYield(dist) of the foe (vehicle.cpp:284-287)
constexpr int NF_PASSED = 2;          // dist + len < 0: the foe's tail has cleared the cross (roadnet.cpp:657)
constexpr int NF_CYCLE = 4;           // the foe's committed blocker chain runs into a cycle (Floyd, roadnet.cpp:662-674)

struct __align__(16) Tail {  // last vehicle of a drivable (Drivable::getLastVehicle), pos < 0 when empty
    double dis, len, speed;
    int pos, prev;
};

struct Ctrl {
    int step;        // Engine::step
    int active;      // activeVehicleCount
    int moverCount;
    int finCount;
    int error;
    int ties;        // same-step entrants of one drivable with EQUAL new distance: their order is unspecified in the
                     // reference (non-stable std::sort over a thread-interleaved buffer, engine.cpp:480); here: priority
    int nVeh[2];     // work lists, double-buffered on step parity
    int nAct[2];
    int nExtra;
    int nBlkUpd;     // sharded mode: blocker changes of this step (see blkUpd)
    int nCustom;     // outstanding set_vehicle_speed requests (Vehicle::setCustomSpeed, vehicle.h:128)
    int epoch;       // steps completed since the engine was created (never reset): stamps the seam messages (device_shard.cuh)
    unsigned long long vehicleSteps;  // sum over steps of activeVehicleCount after the step (the bench metric)
    unsigned long long dbg[8];        // CFB_DEBUG_COUNTERS builds: in-kernel cycle / trip-count maxima
};

#ifdef CFB_DEBUG_COUNTERS
// (per-vehicle cycle / path samples of k_control are recorded in this build: tools/dbg_control_cycles.py)
#endif

}  // namespace cfb
#include "device_lc_types.cuh"
namespace cfb {

constexpr int HEAD_BIT = 0x40000000;   // in vehList[].y: the vehicle is the first of its drivable's list
constexpr int ENT_CAP = 16;   // entrants staged per drivable per step (measured at most 6 on tests/edgenet.py's shapes, DESIGN §4)
constexpr int PLAN_LOOKAHEAD_END = -1;
constexpr int SPAWN_SMEM = 2048;

struct View {
    int nLanes, nLinks, nDrv, nInter, nRL, nCross;
    int moverCap, finCap, vehCap;
    double dt;
    int rl;
    int par;   // step parity (host-provided; equals ctrl->step & 1): selects the live work lists
    // static topology
    const double *drvLength, *drvMaxSpeed;
    const int *off;
    const int *laneOutBeg, *laneOutLinks;
    const int *llStartLane, *llEndLane, *llRoadLink;
    const int4 *linkInfo;   // per laneLink {roadLink, endLane, crossBeg, turn | type << 8}
    const int *llCrossBeg, *lcIdx;
    const double *lcDist;
    const int *csLink;
    const int *interPhaseBeg, *interRLBeg, *phaseAvailBeg, *rlInter;
    const double *phaseTime;
    const unsigned char *phaseAvail, *interVirtual;
    const DTmpl *tmpl;
    const int *planBeg, *planData;
    // dynamic, per position
    double2 *kin, *nkin;
    double *gap;
    int *leader;
    int4 *ids, *nav;
    int2 *nbuf;
    // dynamic, per drivable / slot / cross / intersection
    int *count, *pos;
    int *waitHead, *waitTail, *waitNext;
    int4 *slotInfo;
    unsigned char *inserted;
    Notify *notify;
    Tail *tail;
    unsigned *foeMask;   // per laneLink, maskWords words: crosses of the link whose foe side was notified this step
    const int *lcPeer;   // flat index of the same cross in the other laneLink's cross list
    int maskWords;
    int *curPhase;
    double *remain;
    unsigned char *rlAvail;
    // movers
    int *entCnt, *ent;
    double2 *mkin;
    int4 *mids, *mnav;
    int2 *finSlots;
    // work lists
    int2 *vehList[2];   // {position, drivable} of every running vehicle
    int *actList[2];    // occupied drivables
    int *extraList;     // empty drivables that receive entrants this step
    double *cust;        // per position: custom speed for the coming step (NaN = none)
    double *slotCust;    // per slot: custom speed of a vehicle still in a waiting queue
    int *blk;            // per slot: committed blocker slot (Vehicle::blocker), -1 none: chain walks need one load per hop
    int *delStep;        // per slot: step at which the vehicle in that slot left the network
    // ---- sharded mode (partition.h): null / 0 when the engine owns the whole network ----
    const unsigned char *owned;   // per drivable: 1 = this rank owns it, 2 = a lane it feeds (ghost copy kept in step), 0 = foreign
    const int *ingLanes, *ingLinks, *ingRL;   // k_ingest's index lists: lanes owned or fed, laneLinks / roadLinks owned
    int nIngLanes, nIngLinks, nIngRL;         // (a rank's per-step work must not grow with the size of the WHOLE network)
    const int *boundOut;          // lanes this rank feeds but does not own (all peers, concatenated)
    const int *boundIn;           // lanes this rank owns but a peer feeds
    int nBoundOut, nBoundIn;
    int2 *blkUpd;                 // [0] = {count, 0}; then (slot, new blocker | -2 = left the network)
    int blkUpdCap;
    unsigned *dbgCyc, *dbgPath;   // CFB_DEBUG_COUNTERS builds: per-position cycles / path bits of k_control
    Ctrl *ctrl;
    int *hostMirror;            // pinned, host-mapped: {epoch, active, error, ties} written by k_leader at the end of every step
    const SpawnRec *spawn;      // this step's records (lane-sorted); spawn[-1].slot holds their number
    int lcOn;                   // "laneChange": true
    LcView lc;
};

// ------------------------------------------------------------------------------------------
// Scalar helpers.  The reference is compiled for x86-64 without FMA; conversions double->int
// use cvttsd2si, which yields INT_MIN when out of range (CUDA would saturate).
__device__ __forceinline__ double min2(double x, double y) { return x < y ? x : y; }  // utility.h:70
__device__ __forceinline__ double max2(double x, double y) { return x > y ? x : y; }  // utility.h:66
__device__ __forceinline__ int x86int(double x) {
    return (x > -2147483649.0 && x < 2147483648.0) ? (int) x : INT_MIN;
}
constexpr double kEps = 1e-8;
// Engine::getLaneWaitingVehicleCount engine.cpp:636-648: a vehicle slower than 0.1 m/s is waiting
__device__ __forceinline__ bool isWaiting(double speed) { return speed < 0.1; }
// RoadLink::isAvailable roadnet.h:429-431: roadLink r is available in its intersection's current phase (View::curPhase)
__device__ __forceinline__ unsigned char roadLinkAvailable(const View &V, int r) {
    const int in = V.rlInter[r];
    const int ph = V.interPhaseBeg[in] + V.curPhase[in];
    return V.phaseAvail[V.phaseAvailBeg[ph] + (r - V.interRLBeg[in])];
}

// Vehicle::getNoCollisionSpeed vehicle.cpp:200-209
__device__ __forceinline__ double noCollisionSpeed(double vL, double dL, double vF, double dF, double gap, double dt,
                                                   double targetGap) {
    double c = vF * dt / 2 + targetGap - 0.5 * vL * vL / dL - gap;
    double a = 0.5 / dF;
    double b = 0.5 * dt;
    if (b * b < 4 * a * c) return -100;
    double v1 = 0.5 / a * (sqrt(b * b - 4 * a * c) - b);
    double v2 = 2 * vL - dL * dt + 2 * (gap - targetGap) / dt;
    return min2(v1, v2);
}
// Vehicle::getBrakeDistanceAfterAccel vehicle.cpp:302-306 + getStopBeforeSpeed :240-250
__device__ __forceinline__ double stopBeforeSpeed(const DTmpl &T, double speed, double distance, double dt) {
    double nextSpeed = speed + T.usualPosAcc * dt;
    double brake = (speed + nextSpeed) * dt / 2 + (nextSpeed * nextSpeed / T.usualNegAcc / 2);
    if (brake < distance) return speed + T.usualPosAcc * dt;
    double takeInterval = 2 * distance / (speed + kEps) / dt;
    if (takeInterval >= 1) return speed - speed / x86int(takeInterval);
    return speed - speed / takeInterval;
}
// Vehicle::getDistanceUntilSpeed vehicle.cpp:275-282
__device__ __forceinline__ double distanceUntilSpeed(double mySpeed, double speed, double acc, double dt) {
    if (speed <= mySpeed) return 0;
    int stage1steps = x86int(floor((speed - mySpeed) / acc / dt));
    double stage1speed = mySpeed + stage1steps * acc / dt;
    double stage1dis = (mySpeed + stage1speed) * (stage1steps * dt) / 2;
    return stage1dis + (stage1speed < speed ? ((stage1speed + speed) * dt / 2) : 0);
}
// Vehicle::getReachSteps vehicle.cpp:252-268
__device__ __forceinline__ int reachSteps(double mySpeed, double distance, double targetSpeed, double acc, double dt) {
    if (distance <= 0) return 0;
    if (mySpeed > targetSpeed) return x86int(ceil(distance / mySpeed));
    double du = distanceUntilSpeed(mySpeed, targetSpeed, acc, dt);
    if (du > distance) return x86int(ceil((sqrt(mySpeed * mySpeed + 2 * acc * distance) - mySpeed) / acc / dt));
    return x86int(ceil((targetSpeed - mySpeed) / acc / dt) + ceil((distance - du) / targetSpeed / dt));
}
// Vehicle::canYield vehicle.cpp:284-287
__device__ __forceinline__ bool canYield(const DTmpl &T, double speed, double dist) {
    return (dist > 0 && 0.5 * speed * speed / T.maxNegAcc < dist - T.yieldDistance) || (dist < 0 && dist + T.len < 0);
}

}  // namespace cfb
