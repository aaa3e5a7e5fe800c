// TEST INFRASTRUCTURE ONLY -- what lies ahead of every vehicle in the UNMODIFIED reference engine.
//
// Built by oracle/refctx.mk against the reference sources where they lie under /root/reference (never copied into this
// repository): oracle/_ref/refctx from the unmodified build, oracle/_ref/refctx_lcorder from the priority-ordered copy
// refdump_lcorder is built from (lc_order_patch.sh).  The binaries stay in oracle/_ref/ (git-ignored).
//
//   refctx <config.json> <steps> <threads> <out.bin>
//
// After every step, for every running vehicle (lane-change shadows included) in vehiclePool order:
//   priority, drivable (the static dump's numbering: lanes, then laneLinks), next, signal   4 x int32
//   distance, speed                                                                          2 x double (raw bits)
// next: Router::getNextDrivable() as a drivable index; where there is none, -1 on the route's last road and -2 on a
// lane that cannot continue the route (Router::onValidLane() false).  signal: for a vehicle on a lane whose next
// drivable is a laneLink, RoadLink::isAvailable() of that laneLink's roadLink (0 / 1); else -1.
// getNextDrivable() memoises into Router::planned; the distance and speed are dumped so that a test can check the run
// against `refdump run` / `runlc` step by step: these calls must not change its course.
// File: 'CFC1' | per step: step, n, n records.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <vector>
#include <unistd.h>

#define private public
#define protected public
#include "engine/engine.h"
#undef private
#undef protected

using namespace CityFlow;

int main(int argc, char **argv) {
    if (argc < 5) {
        fprintf(stderr, "usage: refctx <config.json> <steps> <threads> <out.bin>\n");
        return 64;
    }
    Engine e(argv[1], atoi(argv[3]));
    const int steps = atoi(argv[2]);
    std::map<const Drivable *, int32_t> index;
    int32_t k = 0;
    for (Lane *l : e.roadnet.getLanes()) index[l] = k++;
    for (LaneLink *l : e.roadnet.getLaneLinks()) index[l] = k++;
    FILE *fp = fopen(argv[4], "wb");
    if (!fp) { perror(argv[4]); return 2; }
    auto i32 = [fp](int32_t v) { fwrite(&v, 4, 1, fp); };
    auto f64 = [fp](double v) { fwrite(&v, 8, 1, fp); };
    i32(0x43464331);   // 'CFC1'
    for (int s = 0; s < steps; ++s) {
        e.nextStep();
        std::vector<Vehicle *> run;
        for (const auto &vp : e.vehiclePool)
            if (vp.second.first->isRunning()) run.push_back(vp.second.first);
        i32(s + 1);
        i32((int32_t) run.size());
        for (Vehicle *v : run) {
            const Router &router = v->controllerInfo.router;
            Drivable *nd = router.getNextDrivable();
            const int32_t next = nd ? index.at(nd) : (router.onLastRoad() ? -1 : -2);
            int32_t signal = -1;
            if (v->getCurDrivable()->isLane() && nd && nd->isLaneLink())
                signal = static_cast<LaneLink *>(nd)->getRoadLink()->isAvailable() ? 1 : 0;
            i32(v->getPriority());
            i32(index.at(v->getCurDrivable()));
            i32(next);
            i32(signal);
            f64(v->getDistance());
            f64(v->getSpeed());
        }
    }
    // The reference's ~Engine (engine.cpp:762-771) can fail to return when worker threads are still parked on its
    // barriers: the dump is complete, so close it and leave without the destructor (as refdump does).
    fclose(fp);
    fflush(stdout);
    _exit(0);
}
