// device_sim_emu_vehobs.cpp -- the emulated device (tests/device_sim_emu.cpp, included whole) plus the two entry points
// of the per-vehicle table and the batched custom speed, DeviceSim::observeVehicles / setCustomSpeedsFromDevice, run
// with the product's kernel bodies (csrc/device_vehobs.cuh) on the emulated warp.  TEST INFRASTRUCTURE ONLY: built by
// tests/test_cpu_vehicle_obs.py into a library of its own.  The buffers are laid out as
// device_sim.cu lays them out; "device memory" is host memory here, so a caller reads the pointers directly.
#include "device_sim_emu.cpp"

// the atomics device_vehobs.cuh uses, on the one OS thread of the emulated warp
static inline int atomicExch(int *p, int v) { int o = *p; *p = v; return o; }
static inline unsigned long long atomicExch(unsigned long long *p, unsigned long long v) { unsigned long long o = *p; *p = v; return o; }
static inline long long __double_as_longlong(double d) { long long v; memcpy(&v, &d, 8); return v; }
#include "device_vehobs.cuh"

namespace cfb {

struct VehObsEmu {   // what DeviceSim::Impl holds for the two entry points in device_sim.cu
    cfbtest::Buf<int> ints, stamp;
    cfbtest::Buf<double> dbl;
    cfbtest::Buf<unsigned char> shadow;
    VehObsTable T{};
    int tiles = 0, call = 0;
};
// per engine, like g_shardEmu.  An engine made at a freed engine's address inherits its entry, which is harmless: the table
// is re-laid out when its size differs and every refresh rewrites the rows in use and re-pads the ones before; stamps of
// earlier calls are below the next call's number.
static std::map<const DeviceSim::Impl *, VehObsEmu> g_vehObsEmu;

DeviceVehObs DeviceSim::observeVehicles(void *) {
    HostSim &H = impl_->H;
    if (H.V.owned) throw std::runtime_error("observeVehicles: not available on one rank of a sharded run");
    VehObsEmu &E = g_vehObsEmu[impl_];
    const size_t cap = (size_t) std::max(H.P, 1), nD = (size_t) H.V.nDrv;
    const int tiles = (int) std::max<size_t>(1, (nD + blockDim.x - 1) / blockDim.x);
    const size_t nI = 3 * cap + (nD + 1) + 2 + (size_t) tiles;
    if (E.ints.size() != nI || E.tiles != tiles) {
        E.ints.assign(nI, 0);
        std::fill(E.ints.begin(), E.ints.begin() + cap, -1);
        E.dbl.assign(2 * cap, 0.0);
        E.shadow.assign(cap, 0);
        VehObsTable &T = E.T;
        T.slot = E.ints.p(); T.priority = T.slot + cap; T.drivable = T.priority + cap;
        T.drvBegin = T.drivable + cap; T.count = T.drvBegin + nD + 1; T.prevCount = T.count + 1; T.tileSum = T.prevCount + 1;
        T.distance = E.dbl.p(); T.speed = E.dbl.p() + cap; T.shadow = E.shadow.p();
        E.tiles = tiles;
    }
    const View &V = H.V;
    const VehObsTable &T = E.T;
    H.run(E.tiles, [&](int b, int) { vobsTileSums(V, T, b); });
    H.run(E.tiles, [&](int b, int nb) { vobsFill(V, T, b, nb); });
    launches_ += 2;
    DeviceVehObs o;
    o.slot = T.slot; o.priority = T.priority; o.drivable = T.drivable;
    o.distance = T.distance; o.speed = T.speed; o.shadow = T.shadow;
    o.drivableBegin = T.drvBegin; o.count = T.count;
    o.capacity = (long long) cap;
    o.nDrv = H.V.nDrv;
    o.device = -1;
    return o;
}

void DeviceSim::setCustomSpeedsFromDevice(const int32_t *slot, const int32_t *priority, const double *speed, long long n, void *) {
    HostSim &H = impl_->H;
    if (H.V.owned) throw std::runtime_error("setCustomSpeedsFromDevice: not available on one rank of a sharded run");
    if (n < 0 || n > INT_MAX) throw std::runtime_error("setCustomSpeedsFromDevice: entry count out of range");
    VehObsEmu &E = g_vehObsEmu[impl_];
    if (E.stamp.size() < (size_t) H.slotCap) { E.stamp.assign((size_t) H.slotCap, 0); E.call = 0; }
    if (++E.call == INT_MAX) { std::fill(E.stamp.begin(), E.stamp.end(), 0); E.call = 1; }
    if (n == 0) return;
    const int grid = (int) ((n + blockDim.x - 1) / blockDim.x);
    H.run(grid, [&](int b, int nb) { vspeedApply(H.V, slot, priority, speed, (int) n, E.stamp.p(), H.slotCap, E.call, b, nb); });
    launches_ += 1;
}

DeviceVehObs observeVehiclesOf(DeviceSim &dev, void *consumerStream) { return dev.observeVehicles(consumerStream); }
void setCustomSpeedsOf(DeviceSim &dev, const int32_t *slot, const int32_t *priority, const double *speed, long long n,
                       void *producerStream) {
    dev.setCustomSpeedsFromDevice(slot, priority, speed, n, producerStream);
}

}  // namespace cfb
