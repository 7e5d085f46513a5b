// extender::UnschedulablePodMarker::DoesPodsExceedClusterCapacity (one gp_exceeds_cluster_capacity call for the whole sweep)
// against the host layer's per-driver path: DoesPodExceedClusterCapacity as the reference runs it -- the metadata of the
// driver's affinity nodes under zero usage, those nodes in (shuffled) lister order as both priority orders, and the
// packer's BinpackFunc -- for all five `binpack:` values.  Random clusters with several zones and affinity classes,
// negative schedulable dimensions, GPU and non-GPU nodes, empty classes, class -1 drivers and counts at the boundary.
// Needs an H100.
#include <algorithm>
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "gangpack_host.hpp"

static int failures = 0;
#define EXPECT(cond, msg)                                                            \
    do {                                                                             \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

using resources::CreateResources;
using resources::NodeGroupSchedulingMetadata;
static const int64_t Gi = 1ll << 30;

static void Trial(std::mt19937_64& rng, const binpacker::Binpacker& packer, int n, int nClasses, int nZones, char* label) {
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    NodeGroupSchedulingMetadata md;
    std::unordered_map<std::string, int32_t> nodeClass;
    std::vector<std::string> names;
    for (int i = 0; i < n; ++i) {
        char buf[16]; std::snprintf(buf, sizeof buf, "n%05d", i);
        names.push_back(buf);
        resources::NodeSchedulingMetadata m;
        int64_t sc = U(1, 32) * 1000 + (U(0, 3) == 0 ? U(0, 999) : 0), sm = U(1, 64) * Gi, sg = U(0, 3) == 0 ? U(1, 4) : 0;
        if (U(0, 19) == 0) sc = -U(1, 2000);                                  // overhead above allocatable
        if (U(0, 29) == 0) sg = -1;
        m.SchedulableResources = m.AvailableResources = CreateResources(sc, sm, sg);   // zero usage
        m.ZoneLabel = U(0, 9) == 0 ? "default" : "zone-" + std::to_string(U(0, nZones - 1));
        md[buf] = m;
        const int32_t c = (int32_t)U(-1, nClasses - 1);
        if (c >= 0) nodeClass[buf] = c;
    }
    std::vector<extender::UnschedulablePodMarker::StaleDriver> drivers;
    for (int q = 0; q < 60; ++q) {
        extender::UnschedulablePodMarker::StaleDriver d;
        d.DriverResources = CreateResources(U(0, 4) * 500, U(0, 4) * Gi, U(0, 5) == 0 ? 1 : 0);
        d.ExecutorResources = U(0, 15) == 0 ? resources::Zero() : CreateResources(U(0, 4) * 1000, U(0, 8) * (Gi / 2), U(0, 5) == 0 ? 1 : 0);
        d.AffinityClass = (int)U(-1, nClasses);                               // nClasses: a class without nodes
        d.MinExecutorCount = (int)U(0, 3 * n);
        drivers.push_back(d);
    }
    const extender::UnschedulablePodMarker marker(packer);
    const std::vector<bool> got = marker.DoesPodsExceedClusterCapacity(md, nodeClass, nClasses + 1, drivers);
    EXPECT(got.size() == drivers.size(), label);
    for (size_t i = 0; i < drivers.size(); ++i) {
        const auto& d = drivers[i];
        std::vector<std::string> nodeNames;
        NodeGroupSchedulingMetadata sub;
        for (const auto& nm : names) {
            auto c = nodeClass.find(nm);
            if (d.AffinityClass == -1 || (c != nodeClass.end() && c->second == d.AffinityClass)) { nodeNames.push_back(nm); sub[nm] = md.at(nm); }
        }
        std::shuffle(nodeNames.begin(), nodeNames.end(), rng);              // lister order is arbitrary
        const binpack::PackingResult r = packer.BinpackFunc(d.DriverResources, d.ExecutorResources, d.MinExecutorCount, nodeNames, nodeNames, sub);
        if (got[i] != !r.HasCapacity) {
            std::snprintf(label + 40, 40, " driver %zu", i);
            EXPECT(false, label);
        }
    }
}

int main() {
    std::mt19937_64 rng(9120);
    for (const char* name : {binpacker::tightlyPack, binpacker::distributeEvenly, binpacker::azAwareTightlyPack,
                             binpacker::SingleAzTightlyPack, binpacker::SingleAzMinimalFragmentation}) {
        const binpacker::Binpacker& p = *binpacker::SelectBinpacker(name);
        for (int n : {5, 40, 300}) {
            char label[96] = {0};
            std::snprintf(label, 40, "%s n=%d", name, n);
            Trial(rng, p, n, 3, 4, label);
        }
    }
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_capacity_check_test: all passed\n");
    return 0;
}
