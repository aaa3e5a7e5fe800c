// Test helper: prints the static tables our host loader derives (hex floats) as JSON.
#include <cstdio>
#include <string>
#include "../cityflow_b200/csrc/json_min.h"
#include "../cityflow_b200/csrc/roadnet.h"
int main(int argc, char **argv) {
    if (argc < 2) return 2;
    bool ok = false;
    cfb::Json cfg = cfb::Json::parseFile(argv[1], &ok);
    cfb::RoadNet n;
    if (!ok || !n.load(cfg.find("dir")->s + cfg.find("roadnetFile")->s)) return 1;
    printf("{\"n_lanes\": %d, \"n_links\": %d, \"n_cross\": %d, \"lane_length\": [", n.nLanes(), n.nLinks(), n.nCross());
    for (int i = 0; i < n.nLanes(); ++i) printf("%s\"%a\"", i ? "," : "", n.laneLength[i]);
    printf("], \"link_length\": [");
    for (int i = 0; i < n.nLinks(); ++i) printf("%s\"%a\"", i ? "," : "", n.llLength[i]);
    printf("], \"crosses\": [");
    bool first = true;
    for (int l = 0; l < n.nLinks(); ++l)
        for (const cfb::CrossRef &c : n.llCrosses[l]) {
            printf("%s[%d,%d,%d,\"%a\",\"%a\"]", first ? "" : ",", c.cross, c.side, n.nLanes() + n.crossLink[1 - c.side][c.cross],
                   n.crossDist[c.side][c.cross], n.crossDist[1 - c.side][c.cross]);
            first = false;
        }
    printf("], \"lane_out\": [");
    for (int l = 0; l < n.nLanes(); ++l) {
        printf("%s[", l ? "," : "");
        for (size_t j = 0; j < n.laneOutLinks[l].size(); ++j) printf("%s%d", j ? "," : "", n.laneOutLinks[l][j]);
        printf("]");
    }
    printf("], \"link_end\": [");
    for (int k = 0; k < n.nLinks(); ++k) printf("%s%d", k ? "," : "", n.llEndLane[k]);
    printf("], \"link_cross_count\": [");
    for (int k = 0; k < n.nLinks(); ++k) printf("%s%d", k ? "," : "", (int) n.llCrosses[k].size());
    printf("]}\n");
    return 0;
}
