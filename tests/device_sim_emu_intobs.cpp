// device_sim_emu_intobs.cpp -- the emulated device (tests/device_sim_emu.cpp, included whole) plus the intersection
// observations, DeviceSim::observeIntersections, run with the product's kernel body (csrc/device_tlobs.cuh) on the
// emulated warp.  TEST INFRASTRUCTURE ONLY: built by tests/test_cpu_intersection_obs.py into a library of its own.  The
// buffers are laid out as device_sim.cu lays them out (IntObsLayout, device_layout.cuh); "device memory" is host
// memory here, so a caller reads the pointers directly.
#include "device_sim_emu.cpp"
#include "device_tlobs.cuh"

namespace cfb {

struct IntObsEmu {   // what DeviceSim::Impl holds for the entry point in device_sim.cu
    cfbtest::Buf<int> tables, ints;
    cfbtest::Buf<double> dbl;
    cfbtest::Buf<unsigned char> mv;
    IntObsTable T{};
    DeviceIntersectionObs out{};
    bool made = false;
};
// per engine, like g_shardEmu.  An engine made at a freed engine's address inherits its entry: the buffers are made
// again when the tables differ, and every refresh rewrites the dynamic columns.
static std::map<const DeviceSim::Impl *, IntObsEmu> g_intObsEmu;

DeviceIntersectionObs DeviceSim::observeIntersections(void *) {
    Impl &I = *impl_;
    HostSim &H = I.H;
    View &V = H.V;
    if (V.owned) throw std::runtime_error("observeIntersections: not available on one rank of a sharded run");
    IntObsEmu &E = g_intObsEmu[impl_];
    const IntObsLayout X = intObsLayout(H.L, V);
    if (!E.made || E.tables != X.ints || E.out.nInter != V.nInter || E.out.nRL != V.nRL) {
        E.tables.assign(X.ints.begin(), X.ints.end());
        const std::vector<int> init = X.initialInts(V);
        E.ints.assign(init.begin(), init.end());
        E.dbl.assign(std::max(V.nInter, 1), 0.0);
        E.mv.assign(X.phaseMovements.begin(), X.phaseMovements.end());
        X.point(E.T, E.tables.p());
        X.pointOut(E.T, E.out, V, E.ints.p(), E.dbl.p(), E.mv.p());
        E.out.device = -1;
        E.made = true;
    }
    if (I.phaseDirty) { for (int i = 0; i < V.nInter; ++i) H.curPhase[i] = I.hPhase[i]; I.phaseDirty = false; }
    const IntObsTable &T = E.T;
    if (T.nTl > 0) {
        H.run((T.nTl + 2) / 3, [&](int b, int nb) { tobsFill(V, T, b, nb); });   // (grid-stride: fewer blocks than warps)
        launches_ += 1;
    }
    return E.out;
}

DeviceIntersectionObs observeIntersectionsOf(DeviceSim &dev, void *consumerStream) { return dev.observeIntersections(consumerStream); }

}  // namespace cfb
