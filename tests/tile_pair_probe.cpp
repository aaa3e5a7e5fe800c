// CPU probe: k_notify and k_move serve two drivables per warp, one per 16-lane tile, and every loop around a warp
// primitive runs to the larger trip count of the two tiles.  TEST INFRASTRUCTURE ONLY.
//
// This is tests/device_step_probe.cpp (the whole device step on the emulated warp, full state against the restatement
// after every step) with one change: right before k_notify and k_move, the work lists are reordered so that the
// tiles of one warp always hold unequal drivables -- the heaviest with the lightest, the second heaviest with the
// second lightest, and so on.  List order does not change results (entrants are rank-sorted, every other output is
// per drivable), so the restatement must still be matched bit for bit.  The probe counts the warps whose tiles had
// different trip counts.
//
//   g++ -std=c++17 -O1 -ffp-contract=off -I/usr/local/cuda/include -Icityflow_b200/csrc tests/tile_pair_probe.cpp \
//       cityflow_b200/csrc/roadnet.cpp cityflow_b200/csrc/flows.cpp -o probe && ./probe config.json steps
#include <algorithm>
#include <vector>

#include "device_hostsim.h"

namespace {

struct PairStats {
    long long notifyPairs = 0, notifyChunksDiffer = 0;     // k_notify: cross chunks of the two tiles' own links
    long long movePairs = 0, moveChunksDiffer = 0;         // k_move: bucket chunks
    long long entrantsDiffer = 0;                          // k_move: one tile sorts entrants, the other has fewer / none
    int maxVehicles = 0, maxCrosses = 0, maxEntrants = 0;  // in a warp whose other tile differs
} g_pairs;

// Heaviest next to lightest, in pairs (2i, 2i + 1) -- the two tiles of one warp in every grid-stride trip.
void interleave(int *list, int n, const std::vector<long long> &weight) {
    std::vector<int> v(list, list + n);
    std::stable_sort(v.begin(), v.end(), [&](int a, int b) { return weight[a] > weight[b]; });
    for (int i = 0, lo = 0, hi = n - 1; lo <= hi; ++i) list[i] = (i & 1) ? v[hi--] : v[lo++];
}

int chunks(int n) { return (n + 15) / 16; }

// Called by every lane of every block: the first lane of block 0 reorders, before any lane reads the list (the lanes
// of the emulated warp run one after the other up to their first warp primitive).
void pairedNotify(cfb::View &V, int b, int nb) {
    if (b == 0 && threadIdx.x == 0) {
        const int n = V.ctrl->nAct[V.par];
        int *list = V.actList[V.par];
        std::vector<long long> w(V.nDrv, 0);
        auto crosses = [&](int d) { return d >= V.nLanes ? V.llCrossBeg[d - V.nLanes + 1] - V.llCrossBeg[d - V.nLanes] : 0; };
        for (int k = 0; k < n; ++k) w[list[k]] = (long long) crosses(list[k]) * 4096 + V.count[list[k]];
        interleave(list, n, w);
        for (int k = 0; k + 1 < n; k += 2) {
            const int a = crosses(list[k]), c = crosses(list[k + 1]);
            ++g_pairs.notifyPairs;
            if (chunks(a) != chunks(c)) {
                ++g_pairs.notifyChunksDiffer;
                g_pairs.maxCrosses = std::max(g_pairs.maxCrosses, std::max(a, c));
            }
        }
    }
    cfb::phase_notify(V, b, nb);
}

void pairedMove(cfb::View &V, int b, int nb) {
    if (b == 0 && threadIdx.x == 0) {
        const int nAct = V.ctrl->nAct[V.par], nExtra = V.ctrl->nExtra;
        std::vector<long long> w(V.nDrv, 0);
        for (int k = 0; k < nAct; ++k) w[V.actList[V.par][k]] = (long long) V.count[V.actList[V.par][k]] * 64 + V.entCnt[V.actList[V.par][k]];
        for (int k = 0; k < nExtra; ++k) w[V.extraList[k]] = V.entCnt[V.extraList[k]];
        interleave(V.actList[V.par], nAct, w);
        interleave(V.extraList, nExtra, w);
        auto item = [&](int k) { return k < nAct ? V.actList[V.par][k] : V.extraList[k - nAct]; };
        for (int k = 0; k + 1 < nAct + nExtra; k += 2) {
            const int a = item(k), c = item(k + 1);
            ++g_pairs.movePairs;
            if (chunks(V.count[a]) != chunks(V.count[c])) {
                ++g_pairs.moveChunksDiffer;
                g_pairs.maxVehicles = std::max(g_pairs.maxVehicles, std::max(V.count[a], V.count[c]));
            }
            if (V.entCnt[a] != V.entCnt[c]) {
                ++g_pairs.entrantsDiffer;
                g_pairs.maxEntrants = std::max(g_pairs.maxEntrants, std::max(V.entCnt[a], V.entCnt[c]));
            }
        }
    }
    cfb::phase_move(V, b, nb);
}

}  // namespace

#define phase_notify(V, b, n) pairedNotify(V, b, n)
#define phase_move(V, b, n) pairedMove(V, b, n)
#define main step_probe_main
#include "device_step_probe.cpp"
#undef main

int main(int argc, char **argv) {
    const int rc = step_probe_main(argc, argv);
    printf("pairs: notify %lld, %lld with different cross chunks (max %d crosses); move %lld, %lld with different bucket chunks "
           "(max %d vehicles), %lld with different entrant counts (max %d entrants)\n",
           g_pairs.notifyPairs, g_pairs.notifyChunksDiffer, g_pairs.maxCrosses, g_pairs.movePairs, g_pairs.moveChunksDiffer,
           g_pairs.maxVehicles, g_pairs.entrantsDiffer, g_pairs.maxEntrants);
    return rc;
}
