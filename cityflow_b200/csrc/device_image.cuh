// device_image.cuh -- the snapshot image of the dynamic state: its region list (one definition for device_sim.cu and
// the emulated device of the tests) and the translation between the image and its decoded form (StateImage,
// device_sim.h) that the reference-schema JSON archive is written from / read into (host_engine.cpp).  Host code only:
// the image is brought to the host / sent to the device by DeviceSim::snapshotToHost / snapshotFromHost + restore, which
// are the same calls the binary archive uses.
//
// Included after device_view.cuh by a DeviceSim implementation (device_sim.cu, tests/device_sim_emu.cpp).
#pragma once
#include <cmath>
#include <cstring>
#include <stdexcept>

namespace cfb {

struct ImageGeometry {
    const int *off;          // host copy of View::off (nDrv + 1 entries)
    int nDrv, nLanes, nInter;
    size_t P;                // positions
};

// (pointer, bytes) of every array a snapshot carries, in image order; slot-indexed arrays last (their size may differ
// between the time a snapshot is taken and the time it is restored).  With lane change on, the per-slot lane-change
// state (LaneChangeInfo + LaneChange, device_lc_types.cuh) is one more of them; everything else of that path is
// rebuilt every step.
inline size_t imageSlotRegions(const View &V) { return V.lcOn ? 7 : 6; }
inline std::vector<std::pair<void *, size_t>> snapshotRegions(const View &V, size_t P, size_t S) {
    const size_t nL = (size_t) std::max(V.nLanes, 1);
    std::vector<std::pair<void *, size_t>> regs = {
        {V.kin, P * sizeof(double2)}, {V.gap, P * sizeof(double)}, {V.leader, P * sizeof(int)},
        {V.ids, P * sizeof(int4)}, {V.nav, P * sizeof(int4)}, {V.cust, P * sizeof(double)},
        {V.count, (size_t) V.nDrv * sizeof(int)}, {V.entCnt, (size_t) V.nDrv * sizeof(int)},
        {V.tail, (size_t) V.nDrv * sizeof(Tail)},
        {V.waitHead, nL * sizeof(int)}, {V.waitTail, nL * sizeof(int)},
        {V.inserted, nL},
        {V.curPhase, (size_t) V.nInter * sizeof(int)}, {V.remain, (size_t) V.nInter * sizeof(double)},
        {V.vehList[0], P * sizeof(int2)}, {V.vehList[1], P * sizeof(int2)},
        {V.actList[0], (size_t) V.nDrv * sizeof(int)}, {V.actList[1], (size_t) V.nDrv * sizeof(int)},
        {V.ctrl, sizeof(Ctrl)},
        {V.pos, S * sizeof(int)}, {V.waitNext, S * sizeof(int)}, {V.slotInfo, S * sizeof(int4)}, {V.slotCust, S * sizeof(double)},
        {V.blk, S * sizeof(int)}, {V.delStep, S * sizeof(int)},
    };
    if (V.lcOn) regs.push_back({V.lc.slot, S * sizeof(LcSlot)});
    return regs;
}

// The serialised image (snapshotToHost): {magic, steps, slotCap, #regions, region bytes...} as long long, then the
// regions, each padded to 256 bytes.
constexpr long long IMAGE_MAGIC = 0x43464241LL;
inline size_t imagePad(size_t b) { return (b + 255) & ~(size_t) 255; }

struct ImageHeader {
    long long steps = 0;
    int slotCap = 0;
    std::vector<size_t> regions;   // bytes of every region
    size_t bytes() const { return (4 + regions.size()) * sizeof(long long); }
    size_t payload() const { size_t t = 0; for (size_t b : regions) t += imagePad(b); return t; }
};
inline ImageHeader imageHeader(long long steps, int slotCap, const std::vector<std::pair<void *, size_t>> &regs) {
    ImageHeader h{steps, slotCap, {}};
    for (auto &r : regs) h.regions.push_back(r.second);
    return h;
}
// out: h.bytes()
inline void writeImageHeader(const ImageHeader &h, unsigned char *out) {
    std::vector<long long> w = {IMAGE_MAGIC, h.steps, (long long) h.slotCap, (long long) h.regions.size()};
    for (size_t b : h.regions) w.push_back((long long) b);
    memcpy(out, w.data(), w.size() * sizeof(long long));
}
// The header of a serialised image of n bytes; throws unless the image is complete.
inline ImageHeader readImageHeader(const unsigned char *data, size_t n) {
    if (n < 4 * sizeof(long long)) throw std::runtime_error("cityflow_b200: truncated archive");
    long long w[4];
    memcpy(w, data, sizeof w);
    if (w[0] != IMAGE_MAGIC) throw std::runtime_error("cityflow_b200: not an archive of this engine");
    ImageHeader h{w[1], (int) w[2], {}};
    const size_t nr = (size_t) w[3];
    if (n < (4 + nr) * sizeof(long long)) throw std::runtime_error("cityflow_b200: truncated archive");
    h.regions.resize(nr);
    for (size_t k = 0; k < nr; ++k) {
        long long b;
        memcpy(&b, data + (4 + k) * sizeof(long long), sizeof b);
        h.regions[k] = (size_t) b;
    }
    if (n < h.bytes() + h.payload()) throw std::runtime_error("cityflow_b200: truncated archive");
    return h;
}
// An image restored into the regions `regs` of an engine (snapshotRegions): the slot-indexed regions may be shorter.
inline void checkImageFits(const ImageHeader &h, const std::vector<std::pair<void *, size_t>> &regs, const View &V) {
    if (h.regions.size() != regs.size()) throw std::runtime_error("cityflow_b200: archive does not match this engine");
    for (size_t k = 0; k < regs.size(); ++k) {
        if (h.regions[k] > regs[k].second) throw std::runtime_error("cityflow_b200: archive does not match this engine (region size)");
        if (k + imageSlotRegions(V) < regs.size() && h.regions[k] != regs[k].second)
            throw std::runtime_error("cityflow_b200: archive was taken on a different road network");
    }
}

// A typed window into a serialised image.  The regions start 232 + k * 256 bytes into the buffer (the header is not a
// multiple of 16 bytes), so the 16-byte-aligned CUDA vector types must not be accessed through pointers of their own type:
// every access is a memcpy of one element.
template <class T> struct ImageSpan {
    unsigned char *p = nullptr;
    T get(size_t i) const { T v; memcpy(&v, p + i * sizeof(T), sizeof(T)); return v; }
    void set(size_t i, const T &v) const { memcpy(p + i * sizeof(T), &v, sizeof(T)); }
};
struct ImageArrays {
    ImageSpan<double2> kin; ImageSpan<double> gap; ImageSpan<int> leader; ImageSpan<int4> ids, nav; ImageSpan<double> cust;
    ImageSpan<int> count, entCnt; ImageSpan<Tail> tail; ImageSpan<int> waitHead, waitTail; ImageSpan<unsigned char> inserted;
    ImageSpan<int> curPhase; ImageSpan<double> remain; ImageSpan<int2> vehList[2]; ImageSpan<int> actList[2];
    ImageSpan<Ctrl> ctrl; ImageSpan<int> pos, waitNext; ImageSpan<int4> slotInfo; ImageSpan<double> slotCust; ImageSpan<int> blk, delStep;
    long long steps; int slotCap;
};

inline std::vector<size_t> imageRegionBytes(const ImageGeometry &G, size_t S) {
    View V{};
    V.nLanes = G.nLanes; V.nDrv = G.nDrv; V.nInter = G.nInter;
    std::vector<size_t> out;
    for (auto &r : snapshotRegions(V, G.P, S)) out.push_back(r.second);
    return out;
}

// Lay the typed pointers over `blob`; checks the header against this engine's geometry.
inline ImageArrays imageMap(unsigned char *blob, size_t n, const ImageGeometry &G) {
    const ImageHeader h = readImageHeader(blob, n);
    ImageArrays A{};
    A.steps = h.steps;
    A.slotCap = h.slotCap;
    if (A.slotCap < 0) throw std::runtime_error("cityflow_b200: corrupt archive (slot capacity)");
    const std::vector<size_t> want = imageRegionBytes(G, (size_t) A.slotCap);
    if (h.regions.size() != want.size()) throw std::runtime_error("cityflow_b200: archive does not match this engine");
    size_t off = h.bytes();
    unsigned char *ptr[32];
    for (size_t k = 0; k < want.size(); ++k) {
        if (h.regions[k] != want[k]) throw std::runtime_error("cityflow_b200: archive was taken on a different road network");
        ptr[k] = blob + off;
        off += imagePad(want[k]);
    }
    int k = 0;
    A.kin.p = ptr[k++]; A.gap.p = ptr[k++]; A.leader.p = ptr[k++]; A.ids.p = ptr[k++];
    A.nav.p = ptr[k++]; A.cust.p = ptr[k++]; A.count.p = ptr[k++]; A.entCnt.p = ptr[k++];
    A.tail.p = ptr[k++]; A.waitHead.p = ptr[k++]; A.waitTail.p = ptr[k++]; A.inserted.p = ptr[k++];
    A.curPhase.p = ptr[k++]; A.remain.p = ptr[k++]; A.vehList[0].p = ptr[k++]; A.vehList[1].p = ptr[k++];
    A.actList[0].p = ptr[k++]; A.actList[1].p = ptr[k++]; A.ctrl.p = ptr[k++];
    A.pos.p = ptr[k++]; A.waitNext.p = ptr[k++]; A.slotInfo.p = ptr[k++]; A.slotCust.p = ptr[k++];
    A.blk.p = ptr[k++]; A.delStep.p = ptr[k++];
    return A;
}

inline void decodeImage(std::vector<unsigned char> &blob, const ImageGeometry &G, StateImage &out) {
    const ImageArrays A = imageMap(blob.data(), blob.size(), G);
    const Ctrl ctrl = A.ctrl.get(0);
    out = StateImage();
    out.step = ctrl.step;
    out.active = ctrl.active;
    out.slotCount = A.slotCap;
    const int lastStep = ctrl.step - 1;
    out.drivables.resize(G.nDrv);
    for (int d = 0; d < G.nDrv; ++d) {
        const int n = A.count.get(d);
        if (n < 0 || n > G.off[d + 1] - G.off[d]) throw std::runtime_error("cityflow_b200: corrupt archive (list length)");
        out.drivables[d].resize(n);
        for (int k = 0; k < n; ++k) {
            const int p = G.off[d] + k;
            StateImage::Running &r = out.drivables[d][k];
            const int4 idv = A.ids.get(p), nv = A.nav.get(p);
            const double2 kin = A.kin.get(p);
            r.slot = idv.x; r.tmpl = idv.y; r.priority = idv.z; r.nextDrivable = idv.w;
            r.planIdx = nv.x; r.prevDrivable = nv.y; r.blockerSlot = nv.z; r.enterLaneLinkTime = nv.w;
            // a blocker that left the network in the last step is dropped lazily on the device (see DeviceSim::debugDump)
            if (r.blockerSlot >= 0 && r.blockerSlot < A.slotCap && A.delStep.get(r.blockerSlot) == lastStep) r.blockerSlot = -1;
            const int lp = A.leader.get(p);
            if (lp >= (int) G.P) throw std::runtime_error("cityflow_b200: corrupt archive (leader)");
            r.leaderSlot = lp >= 0 ? A.ids.get(lp).x : -1;
            r.dis = kin.x; r.speed = kin.y;
            r.gap = lp >= 0 ? A.gap.get(p) : 0.0;
            r.len = 0;
        }
    }
    out.waiting.resize(G.nLanes);
    for (int l = 0; l < G.nLanes; ++l) {
        int guard = 0;
        for (int s = A.waitHead.get(l); s >= 0; s = A.waitNext.get(s)) {
            if (s >= A.slotCap || ++guard > A.slotCap) throw std::runtime_error("cityflow_b200: corrupt archive (waiting queue)");
            const int4 info = A.slotInfo.get(s);
            out.waiting[l].push_back(StateImage::Waiting{s, info.x, info.y, info.z});
        }
    }
    out.curPhase.resize(G.nInter);
    out.remain.resize(G.nInter);
    for (int i = 0; i < G.nInter; ++i) { out.curPhase[i] = A.curPhase.get(i); out.remain[i] = A.remain.get(i); }
}

inline void encodeImage(const StateImage &in, const ImageGeometry &G, std::vector<unsigned char> &blob) {
    if ((int) in.drivables.size() != G.nDrv || (int) in.waiting.size() != G.nLanes || (int) in.curPhase.size() != G.nInter ||
        (int) in.remain.size() != G.nInter)
        throw std::runtime_error("cityflow_b200: archive does not match this road network");
    const size_t S = (size_t) std::max(in.slotCount, 1);
    const ImageHeader h{in.step, (int) S, imageRegionBytes(G, S)};
    blob.assign(h.bytes() + h.payload(), 0);
    writeImageHeader(h, blob.data());
    const ImageArrays A = imageMap(blob.data(), blob.size(), G);
    const int par = (int) (in.step & 1);
    for (size_t p = 0; p < G.P; ++p) { A.leader.set(p, -1); A.cust.set(p, NAN); }
    for (size_t s = 0; s < S; ++s) { A.pos.set(s, -1); A.waitNext.set(s, -1); A.slotCust.set(s, NAN); A.blk.set(s, -1); A.delStep.set(s, INT_MIN); }
    Ctrl c{};
    c.step = (int) in.step;
    c.epoch = (int) in.step;
    c.active = in.active;
    auto slotOk = [&](int s) { return s >= 0 && (size_t) s < S; };
    for (int d = 0; d < G.nDrv; ++d) {
        const auto &L = in.drivables[d];
        const int n = (int) L.size();
        if (n > G.off[d + 1] - G.off[d]) throw std::runtime_error("cityflow_b200: more vehicles on a drivable than its bucket holds");
        A.count.set(d, n);
        Tail t{};
        t.pos = -1; t.prev = -1;
        for (int k = 0; k < n; ++k) {
            const StateImage::Running &r = L[k];
            const int p = G.off[d] + k;
            if (!slotOk(r.slot) || A.pos.get(r.slot) >= 0) throw std::runtime_error("cityflow_b200: corrupt archive (vehicle listed twice)");
            const int blocker = slotOk(r.blockerSlot) ? r.blockerSlot : -1;
            A.pos.set(r.slot, p);
            A.kin.set(p, make_double2(r.dis, r.speed));
            A.ids.set(p, make_int4(r.slot, r.tmpl, r.priority, r.nextDrivable));
            A.nav.set(p, make_int4(r.planIdx, r.prevDrivable, blocker, r.enterLaneLinkTime));
            A.blk.set(r.slot, blocker);
            A.vehList[par].set(c.nVeh[par]++, make_int2(p, k == 0 ? (d | HEAD_BIT) : d));
            if (k == n - 1) { t.dis = r.dis; t.speed = r.speed; t.len = r.len; t.pos = p; t.prev = r.prevDrivable; }
        }
        A.tail.set(d, t);
        if (n > 0) A.actList[par].set(c.nAct[par]++, d);
    }
    for (int d = 0; d < G.nDrv; ++d)   // leaders by position, now that every vehicle has one
        for (size_t k = 0; k < in.drivables[d].size(); ++k) {
            const StateImage::Running &r = in.drivables[d][k];
            const int p = G.off[d] + (int) k;
            if (slotOk(r.leaderSlot) && A.pos.get(r.leaderSlot) >= 0) { A.leader.set(p, A.pos.get(r.leaderSlot)); A.gap.set(p, r.gap); }
        }
    for (int l = 0; l < G.nLanes; ++l) {
        int tail = -1;
        for (const StateImage::Waiting &w : in.waiting[l]) {
            if (!slotOk(w.slot) || A.pos.get(w.slot) >= 0) throw std::runtime_error("cityflow_b200: corrupt archive (waiting vehicle)");
            A.slotInfo.set(w.slot, make_int4(w.tmpl, w.priority, w.plan, 0));
            if (tail < 0) A.waitHead.set(l, w.slot); else A.waitNext.set(tail, w.slot);
            tail = w.slot;
        }
        if (tail < 0) A.waitHead.set(l, -1);
        A.waitTail.set(l, tail);
    }
    if (G.nLanes == 0) { A.waitHead.set(0, -1); A.waitTail.set(0, -1); }
    for (int i = 0; i < G.nInter; ++i) { A.curPhase.set(i, in.curPhase[i]); A.remain.set(i, in.remain[i]); }
    A.ctrl.set(0, c);
}

}  // namespace cfb
