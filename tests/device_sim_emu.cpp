// device_sim_emu.cpp -- class DeviceSim (csrc/device_sim.h) on top of the emulated warp.  TEST INFRASTRUCTURE ONLY.
//
// Links with the REAL host engine (csrc/host_engine.cpp: flows, RNG, slot / priority bookkeeping, C-ABI)
// in place of csrc/device_sim.cu, so that everything above the kernels can be exercised without a GPU:
// tests build oracle/_build/libcfb_hostcheck.so from it and drive it through the same ctypes binding as the
// GPU parity tests.  It is NOT a CPU fallback of the product: it is not part of the package, nothing in
// cityflow_b200/ can load it, and it refuses to construct unless CFB_EMULATED_DEVICE_FOR_TESTS=1 is set.
// The kernel bodies it runs are the product's own headers (csrc/device_*.cuh) on tests/device_emu.h's
// 32-fiber warp -- about a thousand times slower than the GPU.
//
// Implemented: what the single-GPU engine uses (step, lane-change step halves, observations, debug dumps,
// phases, custom speed, plans, reset, snapshots in the product's image format) and the peer-memory seam protocol of
// a loop-back group.  Not emulated (throw): NCCL sharding, device-resident observations / actions, timing.
#include "device_hostsim.h"
#include "device_image.cuh"

#include <stdexcept>

namespace cfb {

using cfbtest::HostSim;

struct DeviceSim::Impl {
    HostSim H;
    DeviceSimOptions opt;
    std::vector<int> hPhase;
    bool phaseDirty = false;
};

// ---- sharding over "peer memory": the ranks of a loop-back group (host_engine.cpp cfb_shard_group_*) live in one process, a
// peer's arena is the other engine's arrays.  Same kernel bodies as on the GPU (device_shard.cuh); what is not emulated is
// the staged NCCL form and everything collective. ----
struct EmuArena {   // what DeviceSim::shardArena() hands out here: where a peer finds this rank's mailboxes
    int *flags, *delStep;
    int2 *blkIn;
    MoverMsg *moverIn;
    TailMsg *tailIn;
    int nIn, nOut;
};
struct ShardEmu {
    int rank = 0, world = 1;
    std::vector<std::vector<int>> bsize;
    std::vector<unsigned char> owned;   // per drivable: 1 = this rank's (debugDump)
    ShardLists lists;
    cfbtest::Buf<int> flags;
    std::vector<int> ints;
    cfbtest::Buf<int2> blkUpd, blkIn;
    cfbtest::Buf<MoverMsg> moverIn;
    cfbtest::Buf<TailMsg> tailIn;
    cfbtest::Buf<ShardPeer> peers;
    EmuArena arena{};
    ShardP2P S{};
    bool connected = false;
};
static std::map<const DeviceSim *, ShardEmu> g_shardEmu;


static void notEmulated(const char *what) { throw std::runtime_error(std::string("device_sim_emu: ") + what + " is not emulated"); }

DeviceSim::DeviceSim(const RoadNet &net, const std::vector<VehicleTemplate> &templates, const Routing &routing, const DeviceSimOptions &opt)
    : impl_(new Impl()) {
    const char *ok = getenv("CFB_EMULATED_DEVICE_FOR_TESTS");
    if (!ok || ok[0] != '1') {
        delete impl_;
        impl_ = nullptr;
        throw std::runtime_error("device_sim_emu: test-only emulated device (set CFB_EMULATED_DEVICE_FOR_TESTS=1); the product has no CPU path");
    }
    Impl &I = *impl_;
    I.opt = opt;
    I.H.init(net, opt.interval, opt.rlTrafficLight, false, cfb::bucketSpacing(templates));
    uploadTemplates(templates);
    uploadPlans(routing);
    reset();
}
DeviceSim::~DeviceSim() {
    g_shardEmu.erase(this);   // (a later engine at the same address must not inherit this one's mailboxes and flags)
    delete impl_;
}

void DeviceSim::uploadTemplates(const std::vector<VehicleTemplate> &templates) {
    HostSim &H = impl_->H;
    for (size_t k = 0; k < templates.size(); ++k) H.tmpl[k] = toDevice(templates[k], impl_->opt.interval);
}
void DeviceSim::uploadPlans(const Routing &routing) { impl_->H.setPlans(routing); }
void DeviceSim::ensureSlotCapacity(int slots) {
    if (getenv("CFB_EMU_HOST_ONLY")) return;
    if (slots > impl_->H.slotCap) throw std::runtime_error("device_sim_emu: slot capacity of the emulated device exceeded");
}
void DeviceSim::uploadLanePlans(const Routing &routing) { impl_->H.setPlans(routing); }
void DeviceSim::enableLaneChange(const RoadNet &, const Routing &routing) {
    impl_->H.V.lcOn = 1;
    uploadLanePlans(routing);
}

void DeviceSim::stageStep(const SpawnRec *recs, int n) {
    Impl &I = *impl_;
    HostSim &H = I.H;
    if ((size_t) n + 1 > H.spawn.size()) H.spawn.resize((size_t) n * 2 + 2);
    H.spawn[0].slot = n;
    for (int k = 0; k < n; ++k) H.spawn[k + 1] = recs[k];
    H.V.spawn = H.spawn.p() + 1;
    if (I.phaseDirty) { for (int i = 0; i < H.V.nInter; ++i) H.curPhase[i] = I.hPhase[i]; I.phaseDirty = false; }
    H.V.par = (int) (steps_ & 1);
}
static const int G = 3;   // blocks per launch (grid-stride loops)
void DeviceSim::step(const SpawnRec *recs, int n) {
    stageStep(recs, n);
    HostSim &H = impl_->H;
    View &V = H.V;
    // Spawner microbenchmark (CFB_EMU_HOST_ONLY=<population>): no kernels; once <population> vehicles are alive the
    // oldest ones "leave" at the rate new ones arrive, so the host's priority table / slot table sit at a steady size.
    static const char *hostOnly = getenv("CFB_EMU_HOST_ONLY");
    if (hostOnly) {
        static std::vector<int> fifo;
        static size_t head = 0;
        const size_t target = (size_t) atol(hostOnly);
        for (int k = 0; k < n; ++k) fifo.push_back(recs[k].slot);
        while (fifo.size() - head > target && H.ctrl.finCount < H.V.finCap) {
            H.finSlots[H.ctrl.finCount++] = make_int2(fifo[head++], (int) steps_);
            H.delStep[0] = 0;
        }
        steps_ += 1;
        return;
    }
    H.run(G, [&](int b, int nb) { phase_ingest(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_notify(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_control(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_move(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_leader(V, b, nb); });
    launches_ += 5;
    steps_ += 1;
}
void DeviceSim::stepLcBegin(const SpawnRec *recs, int n, const int32_t *spare, int nSpare, std::vector<LcShadow> &created) {
    stageStep(recs, n);
    HostSim &H = impl_->H;
    View &V = H.V;
    H.spare.assign(spare, spare + nSpare);
    V.lc.spare = H.spare.p();
    V.lc.nSpare = nSpare;
    H.run(1, [&](int, int) { k_lc_begin(V.lc); });
    H.run(G, [&](int b, int nb) { phase_ingest(V, b, nb); });
    H.run(G, [&](int, int) { k_lc_admitted(V, V.lc); });
    H.run(G, [&](int, int) { k_lc_segments(V, V.lc); });
    H.run(G, [&](int, int) { k_lc_signal(V, V.lc); });
    if (getenv("CITYFLOW_B200_LC_SERIAL")) H.run(1, [&](int, int) { k_lc_schedule(V, V.lc); });
        else {   // the per-road form DeviceSim launches by default
            H.run(1, [&](int, int) { k_lc_order(V, V.lc); });
            H.run(G, [&](int, int) { k_lc_schedule_roads(V, V.lc); });
            H.run(1, [&](int, int) { k_lc_log(V, V.lc); });
        }
    lcCheckCapacity(H.lcCtrl.error);
    created.resize(H.lcCtrl.nShadows);
    for (int k = 0; k < H.lcCtrl.nShadows; ++k) created[k] = LcShadow{H.shadowLog[k].x, H.shadowLog[k].y};
    launches_ += 6;
}
void DeviceSim::stepLcEnd(const int32_t *priorities, int n) {
    HostSim &H = impl_->H;
    View &V = H.V;
    if (n > 0) {
        for (int k = 0; k < n; ++k) H.prio[k] = priorities[k];
        H.run((n + 31) / 32, [&](int, int) { k_lc_priorities(V, V.lc, H.prio.p(), n); });
    }
    H.run(G, [&](int, int) { k_lc_leader(V, V.lc); });
    H.run(G, [&](int b, int nb) { phase_notify(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_control(V, b, nb); });
    if (getenv("CITYFLOW_B200_LC_SERIAL")) H.run(1, [&](int, int) { k_lc_control_tail(V, V.lc); });
    else {
        H.run(1, [&](int, int) { k_lc_tail_order(V, V.lc); });
        H.run(G, [&](int, int) { k_lc_tail_roads(V, V.lc); });
        H.run(1, [&](int, int) { k_lc_tail_clear(V, V.lc); });
    }
    H.run(G, [&](int b, int nb) { phase_move(V, b, nb); });
    H.run(G, [&](int b, int nb) { phase_leader(V, b, nb); });
    launches_ += 6 + (n > 0);
    steps_ += 1;
}
void DeviceSim::synchronize() {}

int DeviceSim::vehicleCount() { return impl_->H.ctrl.active; }
int DeviceSim::errorFlags() { return impl_->H.ctrl.error; }
double DeviceSim::bucketSpacing() const { return impl_->H.L.spacing; }
int DeviceSim::tieCount() { return impl_->H.ctrl.ties; }
void DeviceSim::laneVehicleCount(int32_t *out) { for (int l = 0; l < impl_->H.V.nLanes; ++l) out[l] = impl_->H.count[l]; }
void DeviceSim::laneWaitingVehicleCount(int32_t *out) {
    HostSim &H = impl_->H;
    for (int l = 0; l < H.V.nLanes; ++l) {
        int c = 0;
        for (int k = 0; k < H.count[l]; ++k) c += H.kin[H.L.off[l] + k].y < 0.1;
        out[l] = c;
    }
}
int DeviceSim::runningVehicles(std::vector<SpeedRec> &out) {
    HostSim &H = impl_->H;
    out.clear();
    for (int d = 0; d < H.V.nDrv; ++d)
        for (int k = 0; k < H.count[d]; ++k) {
            const int p = H.L.off[d] + k;
            out.push_back(SpeedRec{H.ids[p].x, d, H.kin[p].y, H.kin[p].x});
        }
    return (int) out.size();
}
int DeviceSim::drainFinished(std::vector<FinRec> &out) {
    HostSim &H = impl_->H;
    const int n = std::min(H.ctrl.finCount, H.V.finCap);
    out.resize(n);
    for (int k = 0; k < n; ++k) out[k] = FinRec{H.finSlots[k].x, H.finSlots[k].y};
    H.ctrl.finCount = 0;
    return n;
}
void DeviceSim::phases(int32_t *out) {
    HostSim &H = impl_->H;
    for (int i = 0; i < H.V.nInter; ++i) out[i] = H.V.rl ? impl_->hPhase[i] : H.curPhase[i];
}
void DeviceSim::setPhase(int intersection, int phase) { impl_->hPhase[intersection] = phase; impl_->phaseDirty = true; }
int DeviceSim::slotDelStep(int slot) { return slot >= 0 && slot < impl_->H.slotCap ? impl_->H.delStep[slot] : INT_MIN; }
int DeviceSim::numPositions() const { return impl_->H.P; }
int DeviceSim::numDrivables() const { return impl_->H.V.nDrv; }
int DeviceSim::device() const { return -1; }
unsigned long long DeviceSim::vehicleSteps() { return impl_->H.ctrl.vehicleSteps; }

void DeviceSim::reset() {
    impl_->H.reset();
    impl_->hPhase.assign(impl_->H.V.nInter, 0);
    impl_->phaseDirty = false;
    steps_ = 0;
}

void DeviceSim::debugDump(std::vector<DebugRec> &out) {
    auto it = g_shardEmu.find(this);   // one rank of a loop-back group: its own drivables only (the rest holds ghost data)
    debugRecords(impl_->H.V, it != g_shardEmu.end() && !it->second.owned.empty() ? it->second.owned.data() : nullptr, out);
}
void DeviceSim::debugDumpLc(std::vector<LcDebugRec> &out) { lcDebugRecords(impl_->H.V, out); }
bool DeviceSim::vehicleState(int slot, VehState &out) {
    HostSim &H = impl_->H;
    if (slot < 0 || slot >= H.slotCap || H.pos[slot] < 0) return false;
    const int p = H.pos[slot];
    out.pos = p; out.drivable = H.L.posDrv[p]; out.planIdx = H.nav[p].x; out.nextDrv = H.ids[p].w; out.dis = H.kin[p].x; out.speed = H.kin[p].y;
    return true;
}
int DeviceSim::leaderSlotOf(int slot) {
    HostSim &H = impl_->H;
    if (slot < 0 || slot >= H.slotCap || H.pos[slot] < 0) return -2;
    const int lp = H.leader[H.pos[slot]];
    return lp < 0 ? -1 : H.ids[lp].x;
}
void DeviceSim::laneVehicleSlots(std::vector<int32_t> &slots, std::vector<int32_t> &laneBeg) {
    HostSim &H = impl_->H;
    laneBeg.assign(H.V.nLanes + 1, 0);
    slots.clear();
    for (int l = 0; l < H.V.nLanes; ++l) {
        for (int k = 0; k < H.count[l]; ++k) slots.push_back(H.ids[H.L.off[l] + k].x);
        laneBeg[l + 1] = (int) slots.size();
    }
}
void DeviceSim::setCustomSpeed(int slot, double speed) {
    HostSim &H = impl_->H;
    double &dst = H.pos[slot] >= 0 ? H.cust[H.pos[slot]] : H.slotCust[slot];
    if (dst != dst) H.ctrl.nCustom += 1;
    dst = speed;
}
void DeviceSim::setVehiclePlan(int slot, int planId, int planIdx, int nextDrv) {
    HostSim &H = impl_->H;
    if (H.pos[slot] >= 0) { H.nav[H.pos[slot]].x = planIdx; H.ids[H.pos[slot]].w = nextDrv; }
    else H.slotInfo[slot].z = planId;
}

void DeviceSim::configureShard(int rank, int world, const std::vector<unsigned char> &owned, const std::vector<std::vector<int>> &feedPerPeer,
                               const std::vector<std::vector<int>> &ownPerPeer, const std::vector<std::vector<int>> &boundarySize,
                               const std::vector<unsigned char> &ownedRoadLinks) {
    ShardEmu &E = g_shardEmu[this];
    View &V = impl_->H.V;
    E.rank = rank; E.world = world; E.bsize = boundarySize; E.owned = owned;
    E.lists = shardLists(V.nLanes, V.nLinks, owned, feedPerPeer, ownPerPeer, ownedRoadLinks);
    V.owned = E.lists.owned.data();
    E.lists.point(V, E.lists.ing.data(), E.lists.boundOut.data(), E.lists.boundIn.data());
    V.blkUpdCap = BLK_IN_CAP;
    E.blkUpd.assign(1 + V.blkUpdCap, make_int2(0, 0));
    V.blkUpd = E.blkUpd.p();
}
DeviceSim::ShardArena DeviceSim::shardArena() {
    ShardEmu &E = g_shardEmu[this];
    HostSim &H = impl_->H;
    if (E.flags.empty()) {
        E.flags.assign((size_t) SHARD_FLAG_KINDS * E.world, 0);
        E.blkIn.assign((size_t) 2 * E.world * (1 + BLK_IN_CAP), make_int2(0, 0));
        E.moverIn.assign((size_t) 2 * std::max(H.V.nBoundIn, 1), MoverMsg{});
        E.tailIn.assign((size_t) 2 * std::max(H.V.nBoundOut, 1), TailMsg{});
        E.arena = EmuArena{E.flags.p(), H.delStep.p(), E.blkIn.p(), E.moverIn.p(), E.tailIn.p(), std::max(H.V.nBoundIn, 1), std::max(H.V.nBoundOut, 1)};
    }
    return ShardArena{&E.arena, sizeof(EmuArena)};
}
void DeviceSim::shardConnect(const std::vector<void *> &peerBase) {
    ShardEmu &E = g_shardEmu[this];
    const int W = E.world, me = E.rank;
    E.peers.assign(W, ShardPeer{});
    for (int q = 0; q < W; ++q) {
        const EmuArena &A = *static_cast<const EmuArena *>(peerBase[q]);
        ShardPeer &P = E.peers[q];
        P.flags = A.flags; P.delStep = A.delStep; P.blkIn = A.blkIn + (size_t) me * (1 + BLK_IN_CAP);
        P.moverIn = A.moverIn; P.tailIn = A.tailIn; P.nIn = A.nIn; P.nOut = A.nOut;
    }
    const SeamIndex X = seamIndex(seamTables(E.bsize, me));
    E.ints = X.ints;
    ShardP2P &S = E.S;
    S.peers = E.peers.p(); S.me = me; S.world = W;
    X.point(S, E.ints.data());
    S.flags = E.flags.p(); S.blkIn = E.blkIn.p(); S.moverIn = E.moverIn.p(); S.tailIn = E.tailIn.p();
    E.connected = true;
}
bool DeviceSim::shardVehicleCount(int *) { return false; }
void DeviceSim::launchForm(int out[4]) const { for (int k = 0; k < 4; ++k) out[k] = 0; }   // no graph, no PDL, no grid, no mirror
void DeviceSim::stepGrids(int out[5]) const { for (int k = 0; k < 4; ++k) out[k] = G; out[4] = 0; }
void DeviceSim::shardStepTimes(double *ms, long long *steps) { for (int k = 0; k < SHARD_PHASES; ++k) ms[k] = 0; if (steps) *steps = 0; }
void DeviceSim::shardMarkArenaExported() {}
// the peer-memory segments of the loop-back group, kernel for kernel as on the GPU
void DeviceSim::shardSegment(int k) {
    ShardEmu &E = g_shardEmu[this];
    if (!E.connected) notEmulated("the staged (NCCL) seam exchange");
    HostSim &H = impl_->H;
    View &V = H.V;
    auto launch = [&](auto body) { H.run(G, body); launches_ += 1; };
    if (k == 0) {
        launch([&](int b, int nb) { phase_ingest(V, b, nb); });
        launch([&](int b, int nb) { phase_notify(V, b, nb); });
        launch([&](int b, int nb) { phase_control(V, b, nb); });
        launch([&](int, int) { sendMoversBody(V, E.S); });
    } else if (k == 1) {
        launch([&](int, int) { recvMoversBody(V, E.S); });
        launch([&](int b, int nb) { phase_move(V, b, nb); });
        launch([&](int, int) { sendTailsBody(V, E.S); });
    } else {
        launch([&](int, int) { recvTailsBody(V, E.S); });
        launch([&](int b, int nb) { phase_leader(V, b, nb); });
        steps_ += 1;
    }
}
void DeviceSim::shardStep(const SpawnRec *, int, ShardTransport *) { notEmulated("the multi-process sharded step"); }
ShardBuffers DeviceSim::shardBuffers() { return ShardBuffers(); }
void DeviceSim::shardCounts(ShardTransport *, int32_t *, int *) { notEmulated("sharding"); }
void DeviceSim::shardWaitingCounts(ShardTransport *, int32_t *) { notEmulated("sharding"); }
void DeviceSim::shardGatherFinished(ShardTransport *, std::vector<FinRec> &) { notEmulated("sharding"); }
DeviceObs DeviceSim::observeOnDevice(void *) { notEmulated("device-resident observations"); return DeviceObs(); }
void DeviceSim::setPhasesFromDevice(const int32_t *, void *) { notEmulated("device-resident actions"); }
// ---- snapshots: the serialised image of device_sim.cu (device_image.cuh), kept on the host ----
struct DeviceSim::Snapshot { std::vector<unsigned char> bytes; };
DeviceSim::Snapshot *DeviceSim::snapshot() {
    Impl &I = *impl_;
    HostSim &H = I.H;
    if (I.phaseDirty) { for (int i = 0; i < H.V.nInter; ++i) H.curPhase[i] = I.hPhase[i]; I.phaseDirty = false; }
    const auto regs = snapshotRegions(H.V, (size_t) H.P, (size_t) H.slotCap);
    const ImageHeader h = imageHeader(steps_, H.slotCap, regs);
    Snapshot *s = new Snapshot();
    s->bytes.assign(h.bytes() + h.payload(), 0);
    writeImageHeader(h, s->bytes.data());
    size_t off = h.bytes();
    for (auto &r : regs) { if (r.second) memcpy(s->bytes.data() + off, r.first, r.second); off += imagePad(r.second); }
    return s;
}
void DeviceSim::restore(const Snapshot *s) {
    Impl &I = *impl_;
    HostSim &H = I.H;
    const ImageHeader h = readImageHeader(s->bytes.data(), s->bytes.size());
    ensureSlotCapacity(h.slotCap);
    const auto regs = snapshotRegions(H.V, (size_t) H.P, (size_t) H.slotCap);
    checkImageFits(h, regs, H.V);
    for (const Fill &f : slotFills(H.V, (size_t) H.slotCap)) memset(f.p, f.byte, f.bytes);
    size_t off = h.bytes();
    for (size_t k = 0; k < regs.size(); ++k) {
        if (h.regions[k]) memcpy(regs[k].first, s->bytes.data() + off, h.regions[k]);
        off += imagePad(h.regions[k]);
    }
    for (int i = 0; i < H.V.nInter; ++i) I.hPhase[i] = H.curPhase[i];
    I.phaseDirty = false;
    for (const Fill &f : scratchFills(H.V)) memset(f.p, f.byte, f.bytes);
    steps_ = h.steps;
}
void DeviceSim::freeSnapshot(Snapshot *s) { delete s; }
void DeviceSim::snapshotToHost(const Snapshot *s, std::vector<unsigned char> &out) { out = s->bytes; }
DeviceSim::Snapshot *DeviceSim::snapshotFromHost(const unsigned char *data, size_t n) {
    readImageHeader(data, n);
    Snapshot *s = new Snapshot();
    s->bytes.assign(data, data + n);
    return s;
}
static ImageGeometry imageGeometry(DeviceSim::Impl &I) {
    return ImageGeometry{I.H.L.off.data(), I.H.V.nDrv, I.H.V.nLanes, I.H.V.nInter, (size_t) I.H.P};
}
void DeviceSim::decodeSnapshot(const Snapshot *s, StateImage &out) {
    std::vector<unsigned char> blob;
    snapshotToHost(s, blob);
    decodeImage(blob, imageGeometry(*impl_), out);
}
DeviceSim::Snapshot *DeviceSim::encodeSnapshot(const StateImage &in) {
    std::vector<unsigned char> blob;
    encodeImage(in, imageGeometry(*impl_), blob);
    return snapshotFromHost(blob.data(), blob.size());
}
void DeviceSim::enableKernelTiming(bool) {}
void DeviceSim::flushL2() {}
void DeviceSim::markTimed() {}
double DeviceSim::collectTimedMs() { return 0; }
void DeviceSim::debugCounters(unsigned long long out[8], bool) { for (int k = 0; k < 8; ++k) out[k] = 0; }
int DeviceSim::debugArrays(unsigned *, unsigned *) { return 0; }
DeviceSim::KernelTimes DeviceSim::kernelTimes() { return KernelTimes(); }

}  // namespace cfb
