// device_sim_emu_vehctx.cpp -- the emulated device with the per-vehicle entry points (tests/device_sim_emu_vehobs.cpp,
// included whole) plus what lies ahead of each row, DeviceSim::observeVehicleContext, run with the product's kernel body
// (csrc/device_vehobs.cuh, vctxFill) on the emulated warp.  TEST INFRASTRUCTURE ONLY: built by
// tests/test_cpu_vehicle_context.py into a library of its own.  The buffers are laid out as device_sim.cu lays them out;
// "device memory" is host memory here, so a caller reads the pointers directly.
#include "device_sim_emu_vehobs.cpp"

namespace cfb {

struct VehCtxEmu {   // what DeviceSim::Impl holds for the entry point in device_sim.cu
    cfbtest::Buf<int> ints;
    cfbtest::Buf<double> gap;
    cfbtest::Buf<signed char> signal;
    VehCtxTable C{};
};
// per engine, like g_vehObsEmu.  An engine made at a freed engine's address inherits its entry: the buffers are made
// again when the capacity differs, and the mark only widens the first refresh's padding pass.
static std::map<const DeviceSim::Impl *, VehCtxEmu> g_vehCtxEmu;

DeviceVehCtx DeviceSim::observeVehicleContext(void *consumerStream) {
    Impl &I = *impl_;
    HostSim &H = I.H;
    View &V = H.V;
    if (V.owned) throw std::runtime_error("observeVehicleContext: not available on one rank of a sharded run");
    VehCtxEmu &E = g_vehCtxEmu[impl_];
    const size_t cap = (size_t) std::max(H.P, 1);
    if (E.ints.size() != 2 * cap + 2) {   // every row counts as filled, so the first refresh writes the padding of all
        E.ints.assign(2 * cap + 2, -1);
        E.ints[2 * cap] = E.ints[2 * cap + 1] = (int) cap;
        E.gap.assign(cap, 0.0);
        E.signal.assign(cap, 0);
        VehCtxTable &C = E.C;
        C.leader = E.ints.p(); C.nextDrivable = C.leader + cap; C.mark = C.nextDrivable + cap; C.par = 0;
        C.gap = E.gap.p(); C.signal = E.signal.p();
    }
    if (I.phaseDirty) { for (int i = 0; i < V.nInter; ++i) H.curPhase[i] = I.hPhase[i]; I.phaseDirty = false; }
    DeviceVehCtx o;
    o.table = observeVehicles(consumerStream);
    const VehObsTable &T = g_vehObsEmu[impl_].T;
    VehCtxTable &C = E.C;
    H.run((int) ((cap + 95) / 96), [&](int b, int nb) { vctxFill(V, T, C, b, nb); });   // (grid-stride: fewer blocks than rows)
    C.par ^= 1;
    launches_ += 1;
    o.leader = C.leader; o.gap = C.gap; o.nextDrivable = C.nextDrivable; o.signal = C.signal;
    o.drivableLength = V.drvLength; o.drivableMaxSpeed = V.drvMaxSpeed; o.linkRoadLink = V.llRoadLink;
    o.nLanes = V.nLanes; o.nLinks = V.nLinks;
    return o;
}

DeviceVehCtx observeVehicleContextOf(DeviceSim &dev, void *consumerStream) { return dev.observeVehicleContext(consumerStream); }

}  // namespace cfb
