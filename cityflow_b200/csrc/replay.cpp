// replay.cpp -- see replay.h.  FP64 expressions follow the reference's operation order
// (utility.cpp:63-80 Point::unit/normal/len/ang, roadnet.cpp:17-28, :396-410, :750-817) and this
// file is built with -ffp-contract=off, so positions, directions and outlines are the same doubles.
#include "replay.h"

#include <algorithm>
#include <charconv>
#include <cmath>

namespace cfb {
namespace {

inline Pt sub(Pt a, Pt b) { return Pt{a.x - b.x, a.y - b.y}; }
inline Pt add(Pt a, Pt b) { return Pt{a.x + b.x, a.y + b.y}; }
inline Pt mul(Pt a, double k) { return Pt{a.x * k, a.y * k}; }
inline double norm(Pt a) { return std::sqrt(a.x * a.x + a.y * a.y); }          // Point::len
inline Pt unit(Pt a) { const double l = norm(a); return Pt{a.x / l, a.y / l}; }  // Point::unit
inline double cross2(Pt a, Pt b) { return a.x * b.y - a.y * b.x; }              // crossMultiply

}  // namespace

namespace {

inline void put(std::string &s, double v) { putJsonNumber(s, v); }

// getPointByDistance(points, dis)  roadnet.cpp:17-28 (+ getLengthOfPoints :30-35)
Pt pointAt(const std::vector<Pt> &p, double dis) {
    double total = 0.0;
    for (size_t i = 0; i + 1 < p.size(); ++i) total += norm(sub(p[i + 1], p[i]));
    dis = std::max(dis, 0.0);   // max2double(dis, 0): dis unless 0 > dis
    if (!(dis < total)) dis = total;   // min2double(x, y) = x < y ? x : y
    if (dis <= 0.0) return p[0];
    for (size_t i = 1; i < p.size(); ++i) {
        const double len = norm(sub(p[i - 1], p[i]));
        if (dis > len) dis -= len;
        else return add(p[i - 1], mul(sub(p[i], p[i - 1]), dis / len));
    }
    return p.back();
}

// Drivable::getDirectionByDistance  roadnet.cpp:400-410
Pt directionAt(const std::vector<Pt> &p, double dis) {
    double remain = dis;
    for (int i = 0; i + 1 < (int) p.size(); ++i) {
        const double len = norm(sub(p[i + 1], p[i]));
        if (remain < len) return unit(sub(p[i + 1], p[i]));
        remain -= len;
    }
    return unit(sub(p[p.size() - 1], p[p.size() - 2]));
}

}  // namespace

ReplayWriter::ReplayWriter(const RoadNet &net) : net_(net) {
    drvPoints_.reserve(net.nDrivables());
    for (int l = 0; l < net.nLanes(); ++l) drvPoints_.push_back(net.lanePoints[l]);
    for (int k = 0; k < net.nLinks(); ++k) drvPoints_.push_back(net.llPoints[k]);
    roadWidth_.resize(net.nRoads());
    for (int r = 0; r < net.nRoads(); ++r) {  // Road::getWidth roadnet.cpp:693-699
        double w = 0;
        for (int l = net.roadLaneBeg[r]; l < net.roadLaneBeg[r + 1]; ++l) w += net.laneWidth[l];
        roadWidth_[r] = w;
    }
}

std::vector<double> ReplayWriter::outline(int in) const {
    // candidate corner points per attached road, then a Graham scan from the lowest point
    const double width = net_.interWidth[in];
    const Pt pos = net_.interPoint[in];
    std::vector<Pt> pts;
    pts.push_back(pos);
    for (int road : net_.interRoads[in]) {
        Pt dir = unit(sub(net_.interPoint[net_.roadEndInter[road]], net_.interPoint[net_.roadStartInter[road]]));
        const Pt nrm{-dir.y, dir.x};                       // Point::normal of the un-flipped direction
        if (net_.roadStartInter[road] == in) dir = Pt{-dir.x, -dir.y};
        const double roadWidth = roadWidth_[road];
        double delta = 0.5 * (width < roadWidth ? width : roadWidth);
        delta = delta > 5 ? delta : 5;
        const Pt a = sub(pos, mul(dir, width));
        const Pt b = sub(a, mul(nrm, roadWidth));
        pts.push_back(a);
        pts.push_back(b);
        if (delta < net_.roadAverageLength(road)) {
            pts.push_back(sub(a, mul(dir, delta)));
            pts.push_back(sub(b, mul(dir, delta)));
        }
    }
    auto lowest = std::min_element(pts.begin(), pts.end(), [](const Pt &a, const Pt &b) { return a.y < b.y; });
    const Pt p0 = *lowest;
    std::vector<Pt> hull{p0};
    pts.erase(lowest);
    // same library sort, same comparator, same input order as roadnet.cpp:795-797: ties fall the same way
    std::sort(pts.begin(), pts.end(), [p0](const Pt &a, const Pt &b) {
        const Pt da = sub(a, p0), db = sub(b, p0);
        return std::atan2(da.y, da.x) < std::atan2(db.y, db.x);
    });
    for (const Pt &pt : pts) {
        Pt p2 = hull.back();
        if (hull.size() < 2) {
            if (pt.x != p2.x || pt.y != p2.y) hull.push_back(pt);
            continue;
        }
        Pt p1 = hull[hull.size() - 2];
        while (hull.size() > 1 && cross2(sub(pt, p2), sub(p2, p1)) >= 0) {
            p2 = p1;
            hull.pop_back();
            if (hull.size() > 1) p1 = hull[hull.size() - 2];
        }
        hull.push_back(pt);
    }
    std::vector<double> flat;
    for (const Pt &p : hull) { flat.push_back(p.x); flat.push_back(p.y); }
    return flat;
}

std::string ReplayWriter::roadnetJson() const {
    std::string s = "{\"static\":{\"nodes\":[";
    for (int i = 0; i < net_.nInter(); ++i) {
        if (i) s.push_back(',');
        s += "{\"id\":";
        putJsonString(s, net_.interId[i]);
        s += ",\"point\":[";
        put(s, net_.interPoint[i].x); s.push_back(','); put(s, net_.interPoint[i].y);
        s += "],\"virtual\":";
        s += net_.interVirtual[i] ? "true" : "false";
        if (!net_.interVirtual[i]) { s += ",\"width\":"; put(s, net_.interWidth[i]); }
        s += ",\"outline\":[";
        const std::vector<double> o = outline(i);
        for (size_t k = 0; k < o.size(); ++k) { if (k) s.push_back(','); put(s, o[k]); }
        s += "]}";
    }
    s += "],\"edges\":[";
    for (int r = 0; r < net_.nRoads(); ++r) {
        if (r) s.push_back(',');
        s += "{\"id\":";
        putJsonString(s, net_.roadId[r]);
        s += ",\"from\":";
        putJsonString(s, net_.interId[net_.roadStartInter[r]]);
        s += ",\"to\":";
        putJsonString(s, net_.interId[net_.roadEndInter[r]]);
        s += ",\"points\":[";
        for (size_t k = 0; k < net_.roadPoints[r].size(); ++k) {
            if (k) s.push_back(',');
            s.push_back('[');
            put(s, net_.roadPoints[r][k].x); s.push_back(','); put(s, net_.roadPoints[r][k].y);
            s.push_back(']');
        }
        s += "],\"nLane\":";
        s += std::to_string(net_.roadNumLanes(r));
        s += ",\"laneWidths\":[";
        for (int l = net_.roadLaneBeg[r]; l < net_.roadLaneBeg[r + 1]; ++l) {
            if (l > net_.roadLaneBeg[r]) s.push_back(',');
            put(s, net_.laneWidth[l]);
        }
        s += "]}";
    }
    s += "]}}";
    return s;
}

void ReplayWriter::putVehicle(std::string &out, const ReplayVehicle &v, Pt pos, int shadowDepth, int dir) const {
    const Pt d = directionAt(drvPoints_[v.drivable], v.dis);
    put(out, pos.x); out.push_back(' ');
    put(out, pos.y); out.push_back(' ');
    put(out, std::atan2(d.y, d.x)); out.push_back(' ');
    if (v.flow == -2) out += "manually_pushed_" + std::to_string(v.index);
    else out += "flow_" + std::to_string(v.flow) + "_" + std::to_string(v.index);
    for (int k = 0; k < shadowDepth; ++k) out += "_shadow";
    out.push_back(' ');
    out += std::to_string(dir);
    out.push_back(' ');
    put(out, v.len); out.push_back(' ');
    put(out, v.width); out.push_back(',');
}

void ReplayWriter::putLights(std::string &out, const int *phase) const {
    out.push_back(';');
    for (int r = 0; r < net_.nRoads(); ++r) {
        const int in = net_.roadEndInter[r];
        if (net_.interVirtual[in]) continue;
        out += net_.roadId[r];
        const int nPhases = net_.interPhaseBeg[in + 1] - net_.interPhaseBeg[in];
        for (int l = net_.roadLaneBeg[r]; l < net_.roadLaneBeg[r + 1]; ++l) {
            if (nPhases <= 1) { out += " i"; continue; }  // Intersection::isImplicitIntersection roadnet.cpp:819
            bool go = true;
            const int gp = net_.interPhaseBeg[in] + phase[in];
            for (int ll : net_.laneOutLinks[l]) {
                const int rl = net_.llRoadLink[ll];
                if (!net_.phaseAvail[net_.phaseAvailBeg[gp] + (rl - net_.interRoadLinkBeg[in])]) { go = false; break; }
            }
            out += go ? " g" : " r";
        }
        out.push_back(',');
    }
}

void ReplayWriter::formatStep(const ReplayVehicle *v, size_t n, const int *phase, std::string &out) const {
    out.clear();
    for (size_t k = 0; k < n; ++k)   // Vehicle::getPoint with offset 0 (vehicle.cpp:82-84); lastLaneChangeDirection 0
        putVehicle(out, v[k], pointAt(drvPoints_[v[k].drivable], v[k].dis), 0, 0);
    putLights(out, phase);
}

void ReplayWriter::formatStepLc(const ReplayVehicleLc *v, size_t n, const int *phase, std::string &out) const {
    constexpr double eps = 1e-8;   // utility.h:15
    out.clear();
    for (size_t k = 0; k < n; ++k) {
        const ReplayVehicle &u = v[k].v;
        const double off = v[k].offset;
        Pt pos = pointAt(drvPoints_[u.drivable], u.dis);
        if (!(std::fabs(off) < eps) && u.drivable < net_.nLanes()) {   // Vehicle::getPoint vehicle.cpp:81-105
            const int next = off > 0 ? u.drivable + 1 : u.drivable - 1;   // lanes of a road are consecutive, by index
            const Pt q = pointAt(drvPoints_[next], u.dis);
            const double pct = (off > 0 ? 2 * off : -2 * off) / (net_.laneWidth[u.drivable] + net_.laneWidth[next]);
            pos = Pt{q.x * pct + pos.x * (1 - pct), q.y * pct + pos.y * (1 - pct)};
        }
        putVehicle(out, u, pos, v[k].shadowDepth, v[k].dir);
    }
    putLights(out, phase);
}

}  // namespace cfb
