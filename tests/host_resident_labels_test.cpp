// affinity::ResidentLabels with the resident MatchRequiredNodeAffinity and UnschedulablePodMarker's affinity sweep over both
// resident tables (each table flushed once, then one gp_match_node_affinity_resident / _label_table call), driven by random
// node add / relabel / delete events, against the per-call host paths (Encode + gp_match_node_affinity, and the
// per-call affinity sweep) on the same nodes.  Includes capacities that double from one, and a table whose device copy is
// replaced behind its back (a reset) so that the next resident call is refused, replayed and answered by the per-call path.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using affinity::Node;
using affinity::Program;
using affinity::Requirement;
using affinity::ResidentLabels;
using affinity::Term;
using extender::ResidentOverheadComputer;
using extender::UnschedulablePodMarker;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

static bool same(const affinity::MatchResult& a, const affinity::MatchResult& b) { return a.Matched == b.Matched && a.Failed == b.Failed; }

int main() {
    std::mt19937_64 rng(41);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    static const char* keys[] = {"zone", "ig", "gpus", "tier", "example.com/pool", "rank"};
    static const char* vals[] = {"a", "b", "c", "7", "-3", "+5", "9223372036854775807", "-9223372036854775808", "9223372036854775808", "x"};
    auto labelsOf = [&]() {
        std::map<std::string, std::string> l;
        for (const char* k : keys) if (pick(3) != 0) l[k] = vals[pick(10)];
        return l;
    };
    std::vector<Program> programs;
    for (int p = 0; p < 10; ++p) {
        Program pr;
        if (pick(4) == 0) pr.NodeSelector["zone"] = vals[pick(3)];
        pr.HasRequired = pick(6) != 0;
        for (int t = 0; t < 1 + pick(2); ++t) {
            Term term;
            const int op = pick(6);
            static const char* ops[] = {"In", "NotIn", "Exists", "DoesNotExist", "Gt", "Lt"};
            Requirement r{pick(8) == 0 ? "ghost" : keys[pick(6)], ops[op], {}};
            if (op < 2) { r.Values.push_back(vals[pick(10)]); r.Values.push_back(pick(2) ? "ghost-value" : vals[pick(10)]); }
            if (op >= 4) r.Values.push_back(pick(2) ? "4" : "0");
            term.MatchExpressions.push_back(r);
            if (pick(5) == 0) term.MatchFields.push_back(Requirement{"metadata.name", "In", {"node-" + std::to_string(pick(30))}});
            pr.Terms.push_back(term);
        }
        programs.push_back(pr);
    }
    ResidentLabels labels(gp_label_table_size{1, 1, 1, 1});
    ResidentOverheadComputer overhead(gp_overhead_table_size{1, 1, 1, 1, 1});
    const UnschedulablePodMarker marker(*binpacker::SelectBinpacker(binpacker::tightlyPack));
    std::map<std::string, std::map<std::string, std::string>> live;
    int serial = 0;
    for (int step = 0; step < 12; ++step) {
        for (int e = 0; e < 12; ++e) {
            const int r = pick(10);
            if (r < 4 || live.empty()) {
                const std::string name = "node-" + std::to_string(serial++);
                live[name] = labelsOf();
                labels.SetNode(Node{name, live[name]});
            } else if (r < 6) {
                auto it = std::next(live.begin(), pick((int)live.size()));
                labels.DeleteNode(it->first);
                live.erase(it);
            } else {
                auto it = std::next(live.begin(), pick((int)live.size()));
                if (r < 8) it->second = labelsOf();
                labels.SetNode(Node{it->first, it->second});
            }
        }
        std::vector<std::string> names;
        std::vector<Node> nodes;
        for (const auto& kv : live) { names.push_back(kv.first); nodes.push_back(Node{kv.first, kv.second}); }
        names.push_back("unlabelled");
        nodes.push_back(Node{"unlabelled", {}});
        if (step == 7) {                                    // the device's table replaced behind the host's back: a refusal
            gangpack::Device& dev = gangpack::Device::Get();
            labels.Flush(dev);
            gp_label_table_size tiny{1, 1, 1, 1};
            dev.check(gp_label_table_reset(dev.ctx(), &tiny), "gp_label_table_reset");
        }
        EXPECT(same(affinity::MatchRequiredNodeAffinity(names, labels, programs), affinity::MatchRequiredNodeAffinity(nodes, programs)));
        // the marker: both tables resident against the per-call sweep over the same labels and zero overhead
        std::vector<UnschedulablePodMarker::CapacityNode> cap;
        resources::NodeGroupSchedulingMetadata md;
        for (const auto& nm : names) {
            const resources::Resources alloc = resources::CreateResources(4000 + pick(8) * 1000, (int64_t)(8 + pick(24)) << 30, 0);
            const std::string zone = "z" + std::to_string(pick(2));
            cap.push_back({nm, alloc, zone});
            resources::NodeSchedulingMetadata m;
            m.SchedulableResources = alloc;
            m.ZoneLabel = zone;
            md[nm] = m;
        }
        std::vector<UnschedulablePodMarker::AffinityStaleDriver> drivers;
        for (int i = 0; i < 40; ++i) {
            UnschedulablePodMarker::AffinityStaleDriver d;
            d.DriverResources = resources::CreateResources(500 * pick(4), (int64_t)pick(4) << 30, 0);
            d.ExecutorResources = resources::CreateResources(1000 * pick(4), (int64_t)pick(8) << 30, 0);
            d.MinExecutorCount = pick(12);
            d.Affinity = pick((int)programs.size());
            drivers.push_back(d);
        }
        if (step == 9) {
            gangpack::Device& dev = gangpack::Device::Get();
            gp_label_table_size tiny{1, 1, 1, 1};
            dev.check(gp_label_table_reset(dev.ctx(), &tiny), "gp_label_table_reset");
        }
        std::vector<bool> errA, errB;
        const std::vector<bool> a = marker.DoesPodsExceedClusterCapacity(cap, overhead, labels, programs, drivers, &errA);
        const std::vector<bool> b = marker.DoesPodsExceedClusterCapacity(md, nodes, programs, drivers, &errB);
        EXPECT(errA == errB);
        for (size_t i = 0; i < drivers.size(); ++i) EXPECT(errA[i] || a[i] == b[i]);
    }
    if (failures) { std::printf("host_resident_labels_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_labels_test: all passed\n");
    return 0;
}
