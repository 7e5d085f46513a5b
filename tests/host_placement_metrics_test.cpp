// metrics::PlacementMetrics (one gp_placement_metrics call) in the C++ host layer against a string-keyed C++ literal of
// ReportInitialDriverExecutorCollocationMetric, ReportInitialNodeCountMetrics and ReportCrossZoneMetric
// (internal/metrics/metrics.go:223-330): name-keyed maps, a missing failure-domain label read as "unknown-zone", and the zone
// map walked in a random order for crossZoneTraffic, as Go iterates it.  Random clusters and placements: repeated nodes,
// the driver among its executors or not, placed nodes outside availableNodes, nodes labelled unknown-zone next to
// unlabelled ones.  Needs an H100.
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

// the literal: what the three reporters emit for one successful placement
static metrics::PlacementMetricsResult Literal(const std::string& driverNodeName, const std::vector<std::string>& executorNodeNames,
                                               const std::vector<metrics::Node>& nodes, std::mt19937_64& rng) {
    metrics::PlacementMetricsResult r;
    r.Reported = true;
    std::map<std::string, bool> executorNodeNamesSet;                               // toExecutorNodeNamesSet
    for (const auto& n : executorNodeNames) executorNodeNamesSet[n] = true;
    const auto hit = executorNodeNamesSet.find(driverNodeName);                 // a Go map read inserts nothing
    if (hit == executorNodeNamesSet.end() || !hit->second) r.CollocationType = "no-collocation";
    else if (executorNodeNamesSet.size() == 1) r.CollocationType = "driver-collocated-with-all-executors";
    else r.CollocationType = "driver-collocated-with-some-executors";
    const int executorCount = (int)executorNodeNames.size();
    if (executorCount > 0) {
        r.NodeCountReported = true;
        r.ExecutorsPerNode = executorCount / (int)executorNodeNamesSet.size();
        r.NodeCount = (int64_t)executorNodeNamesSet.size();
    }
    std::map<std::string, int> numPodsPerNode{{driverNodeName, 1}};
    for (const auto& n : executorNodeNames) numPodsPerNode[n]++;
    std::map<std::string, int> numPodsPerZone;
    for (const auto& n : nodes) {
        auto it = numPodsPerNode.find(n.Name);
        if (it == numPodsPerNode.end()) continue;
        auto z = n.Labels.find(extender::LabelZoneFailureDomain);
        numPodsPerZone[z == n.Labels.end() ? "unknown-zone" : z->second] += it->second;
    }
    const int totalNumPods = executorCount + 1;
    std::vector<std::string> order;                                               // Go's map iteration: any order
    for (const auto& kv : numPodsPerZone) order.push_back(kv.first);
    std::shuffle(order.begin(), order.end(), rng);
    int64_t numPodsInDifferentZone = totalNumPods, crossZoneTraffic = 0;
    for (const auto& z : order) {
        numPodsInDifferentZone -= numPodsPerZone[z];
        crossZoneTraffic += (int64_t)numPodsPerZone[z] * numPodsInDifferentZone;
    }
    r.CrossZonePairs = crossZoneTraffic;
    r.TotalPairs = (int64_t)totalNumPods * (totalNumPods - 1) / 2;
    r.NumberOfZones = (int64_t)numPodsPerZone.size();
    return r;
}

static bool Same(const metrics::PlacementMetricsResult& a, const metrics::PlacementMetricsResult& b) {
    return a.Reported == b.Reported && a.CollocationType == b.CollocationType && a.NodeCountReported == b.NodeCountReported &&
           a.ExecutorsPerNode == b.ExecutorsPerNode && a.NodeCount == b.NodeCount && a.CrossZonePairs == b.CrossZonePairs &&
           a.TotalPairs == b.TotalPairs && a.NumberOfZones == b.NumberOfZones;
}

static void Trial(std::mt19937_64& rng, int n, int n_labels, int kmax, const char* label) {
    auto U = [&](int lo, int hi) { return lo + (int)(rng() % (uint64_t)(hi - lo + 1)); };
    std::vector<metrics::Node> nodes;
    std::vector<std::string> names;
    for (int i = 0; i < n; ++i) {
        char buf[16]; std::snprintf(buf, sizeof buf, "n%05d", i);
        names.push_back(buf);
        metrics::Node m;
        m.Name = buf;
        const int r = U(0, 19);
        if (r == 0) {}                                                            // no zone label
        else if (r == 1) m.Labels[extender::LabelZoneFailureDomain] = "unknown-zone";
        else m.Labels[extender::LabelZoneFailureDomain] = "zone-" + std::to_string(U(0, n_labels - 1));
        m.Labels["kubernetes.io/hostname"] = buf;
        nodes.push_back(m);
    }
    const int outside = n / 10 + 1;                                              // names not in availableNodes
    for (int i = 0; i < outside; ++i) names.push_back("gone-" + std::to_string(i));
    for (int q = 0; q < 40; ++q) {
        binpack::PackingResult r;
        r.HasCapacity = true;
        const int pool = U(1, (int)names.size());                                // small pools repeat nodes
        r.DriverNode = names[(size_t)U(0, pool - 1)];
        const int k = U(0, kmax);
        for (int t = 0; t < k; ++t) r.ExecutorNodes.push_back(U(0, 3) == 0 ? r.DriverNode : names[(size_t)U(0, pool - 1)]);
        const auto got = metrics::PlacementMetrics(r, nodes);
        const auto want = Literal(r.DriverNode, r.ExecutorNodes, nodes, rng);
        EXPECT(Same(got, want), label);
        if (!Same(got, want))
            std::printf("  %s k=%d: got %s %lld/%lld pairs %lld/%lld zones %lld, want %s %lld/%lld pairs %lld/%lld zones %lld\n", label, k,
                        got.CollocationType.c_str(), (long long)got.ExecutorsPerNode, (long long)got.NodeCount, (long long)got.CrossZonePairs,
                        (long long)got.TotalPairs, (long long)got.NumberOfZones, want.CollocationType.c_str(), (long long)want.ExecutorsPerNode,
                        (long long)want.NodeCount, (long long)want.CrossZonePairs, (long long)want.TotalPairs, (long long)want.NumberOfZones);
    }
    EXPECT(!metrics::PlacementMetrics(binpack::EmptyPackingResult(), nodes).Reported, label);
}

int main() {
    std::mt19937_64 rng(4242);
    Trial(rng, 5, 2, 8, "n=5");
    Trial(rng, 200, 3, 40, "n=200");
    Trial(rng, 3000, 6, 3000, "n=3000 (rows above the warp path)");
    Trial(rng, 64, 64, 50, "n=64, a zone per node");
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_placement_metrics_test: all passed\n");
    return 0;
}
