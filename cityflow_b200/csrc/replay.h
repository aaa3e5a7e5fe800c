// replay.h -- the replay log the reference writes with "saveReplay": true (SURVEY 8f-4).
//
// Two files, read by the reference's frontend viewer:
//   roadnetLogFile  {"static": {"nodes": [...], "edges": [...]}}        RoadNet::convertToJson roadnet.cpp:327-394
//   replayLogFile   one line per step: "<x> <y> <angle> <id> <lc> <len> <width>,...;<road> <g|r|i>...,..."
//                                                                      Engine::updateLog engine.cpp:518-554
// Host-side formatting of (a) the static tables and (b) a per-step list of running vehicles
// {drivable, distance, id, length, width} in vehiclePool (priority) order plus the current phase of
// every intersection -- on the GPU engine that list is one gather from device state, in the parity
// tests it comes from the oracle, so this file has no device dependency.
//
// Parity level: NUMERIC.  The reference prints doubles with dtoa_milo, whose digit generation
// reads past the end of its kPow10 table for more than 9 fraction digits (dtoa_milo.h:275): the
// last digit is not a function of the value alone, so byte-identical files are not definable.
// Here doubles are printed in their shortest round-trip form (std::to_chars); every token parses to
// the same double the reference computed (tests compare parsed values).
#pragma once
#include <string>
#include <vector>
#include "roadnet.h"

namespace cfb {

struct ReplayVehicle {
    int drivable;        // lane id, or nLanes + laneLink id
    double dis;          // distance along the drivable
    int flow, index;     // id: flow_<flow>_<index>, flow == -2: manually_pushed_<index>
    double len, width;   // VehicleInfo len / width
};

struct ReplayVehicleLc { // a running vehicle of a lane-change run (cfb_replay_vehicle_lc)
    ReplayVehicle v;
    int shadowDepth;     // "_shadow" suffixes of the id
    int dir;             // LaneChange::lastDir
    double offset;       // LaneChangeInfo::offset
};

// JSON output pieces (json_write.cpp).  putJsonNumber: the shortest digit string that parses back to `v`, laid out like
// the reference's printer ("2.0", "12.34", "1.234e33").  putJsonNumberLikeRapidjson: the digits rapidjson's writer
// (Grisu2) emits -- the archive writer uses it so that the reference reads back the doubles it would from its own file.
void putJsonNumber(std::string &s, double v);
void putJsonNumberLikeRapidjson(std::string &s, double v);
void putJsonString(std::string &s, const std::string &v);

class ReplayWriter {
public:
    explicit ReplayWriter(const RoadNet &net);
    // roadnetLogFile content (no trailing newline)
    std::string roadnetJson() const;
    // one replayLogFile line (no trailing newline).  vehicles: running vehicles in ascending
    // priority; phase[i]: current phase index of intersection i (ignored for virtual ones).
    void formatStep(const ReplayVehicle *vehicles, size_t n, const int *phase, std::string &out) const;
    // the same with lane change: off-centre positions, suffixed ids, change directions
    void formatStepLc(const ReplayVehicleLc *vehicles, size_t n, const int *phase, std::string &out) const;
    // Intersection::getOutline roadnet.cpp:750-817 (flattened x0,y0,x1,y1,...)
    std::vector<double> outline(int intersection) const;

private:
    void putVehicle(std::string &out, const ReplayVehicle &v, Pt pos, int shadowDepth, int dir) const;
    void putLights(std::string &out, const int *phase) const;
    const RoadNet &net_;
    std::vector<std::vector<Pt>> drvPoints_;      // lanes then laneLinks
    std::vector<double> roadWidth_;
};

}  // namespace cfb
