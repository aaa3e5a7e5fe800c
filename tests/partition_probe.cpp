// Test helper: prints the partition of a scenario as JSON -- column strips, or the cut given as a comma-separated list of
// intersection owners (Partition::fromOwners, what cfb_debug_shard_group_create_cut builds).
// Usage: partition_probe <config> <world> [<rank> | -1] [<owner>,<owner>,...]
#include <cstdio>
#include <cstdlib>
#include <string>
#include "../cityflow_b200/csrc/json_min.h"
#include "../cityflow_b200/csrc/partition.h"
int main(int argc, char **argv) {
    if (argc < 3) return 2;
    bool ok = false;
    cfb::Json cfg = cfb::Json::parseFile(argv[1], &ok);
    cfb::RoadNet n;
    if (!ok || !n.load(cfg.find("dir")->s + cfg.find("roadnetFile")->s)) return 1;
    const int world = atoi(argv[2]);
    cfb::Partition p;
    if (argc >= 5) {
        std::vector<int> owner;
        for (const char *c = argv[4]; *c;) {
            char *end = nullptr;
            owner.push_back((int) strtol(c, &end, 10));
            c = *end ? end + 1 : end;
        }
        if ((int) owner.size() != n.nInter()) return 3;
        for (int o : owner) if (o < 0 || o >= world) return 3;
        p = cfb::Partition::fromOwners(n, owner, world);
    } else {
        p = cfb::Partition::columnStrips(n, world);
    }
    printf("{\"world\": %d, \"n_lanes\": %d, \"inter_owner\": [", world, n.nLanes());
    for (int i = 0; i < n.nInter(); ++i) printf("%s%d", i ? "," : "", p.interOwner[i]);
    printf("], \"inter_virtual\": [");
    for (int i = 0; i < n.nInter(); ++i) printf("%s%d", i ? "," : "", (int) n.interVirtual[i]);
    printf("], \"lane_owner\": [");
    for (int l = 0; l < n.nLanes(); ++l) printf("%s%d", l ? "," : "", p.drvOwner[l]);
    printf("], \"lane_feeder\": [");
    for (int l = 0; l < n.nLanes(); ++l) printf("%s%d", l ? "," : "", p.interOwner[n.roadStartInter[n.laneRoad[l]]]);
    printf("], \"lane_start\": [");
    for (int l = 0; l < n.nLanes(); ++l) printf("%s%d", l ? "," : "", n.roadStartInter[n.laneRoad[l]]);
    printf("], \"lane_end\": [");
    for (int l = 0; l < n.nLanes(); ++l) printf("%s%d", l ? "," : "", n.roadEndInter[n.laneRoad[l]]);
    printf("], \"boundary\": [");
    for (int a = 0; a < world; ++a) {
        printf("%s[", a ? "," : "");
        for (int b = 0; b < world; ++b) {
            printf("%s[", b ? "," : "");
            for (size_t k = 0; k < p.boundary[a][b].size(); ++k) printf("%s%d", k ? "," : "", p.boundary[a][b][k]);
            printf("]");
        }
        printf("]");
    }
    printf("]");
    if (argc >= 4 && atoi(argv[3]) >= 0) {   // seam tables of one rank (what DeviceSim::shardConnect uploads), with the rank's own lane lists
        const int me = atoi(argv[3]);
        std::vector<std::vector<int>> bsize(world, std::vector<int>(world, 0));
        for (int a = 0; a < world; ++a) for (int b = 0; b < world; ++b) bsize[a][b] = (int) p.boundary[a][b].size();
        const cfb::SeamTables t = cfb::seamTables(bsize, me);
        auto arr = [](const char *name, const std::vector<int> &v) {
            printf(", \"%s\": [", name);
            for (size_t k = 0; k < v.size(); ++k) printf("%s%d", k ? "," : "", v[k]);
            printf("]");
        };
        std::vector<int> outLanes, inLanes;   // the order DeviceSim::configureShard lists them in
        for (int q = 0; q < world; ++q) {
            outLanes.insert(outLanes.end(), p.boundary[me][q].begin(), p.boundary[me][q].end());
            inLanes.insert(inLanes.end(), p.boundary[q][me].begin(), p.boundary[q][me].end());
        }
        arr("nbr", t.nbr); arr("out_peer", t.outPeer); arr("out_dst", t.outDst); arr("in_peer", t.inPeer); arr("in_dst", t.inDst);
        arr("out_lanes", outLanes); arr("in_lanes", inLanes);
    }
    printf(", \"validate\": \"%s\"}\n", p.validate(n, 64.2).c_str());
    return 0;
}
