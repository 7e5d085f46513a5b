// extender::ReconcileFindNodesNodeTable and UnschedulablePodMarker's node-table sweeps (the C++ host layer of
// gp_reconcile_find_nodes_node_table and gp_exceeds_cluster_capacity[_affinity]_node_table), driven by random node add /
// update / delete events over resources::ResidentNodes (with creation times, some equal), affinity::ResidentLabels,
// extender::ResidentReservations and an extender::ResidentOverheadComputer.  After every round each node-table path must
// equal the resident path given the columns the host keeps itself (allocatable, flags, creation and the label strings):
// ReconcileFindNodesResident and the resident marker sweeps.  An instance-group value left out of the list, and a node table
// replaced behind the host's back (a reset), make the device call refuse; the host path then replays and still answers.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using affinity::Node;
using affinity::Program;
using affinity::ResidentLabels;
using extender::ReconcileNode;
using extender::ReconcileResult;
using extender::ResidentOverheadComputer;
using extender::ResidentReservations;
using extender::UnschedulablePodMarker;
using resources::NodeTableLabels;
using resources::ResidentNodes;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

static bool same(const std::vector<ReconcileResult>& a, const std::vector<ReconcileResult>& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if (a[i].InstanceGroupFound != b[i].InstanceGroupFound || a[i].ReservedNodeNames != b[i].ReservedNodeNames) return false;
    return true;
}

struct Host {                              // what the host knows of a node, kept beside the tables
    std::map<std::string, std::string> labels;
    resources::Resources alloc;
    bool unschedulable = false, ready = true;
    int64_t creation = 0;
};

int main() {
    std::mt19937_64 rng(91);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    gangpack::Device& dev = gangpack::Device::Get();
    ResidentLabels labels(gp_label_table_size{1, 1, 1, 1});
    ResidentNodes nodes(labels, 1, 10);
    ResidentReservations reservations(gp_reservation_table_size{1, 1});
    ResidentOverheadComputer overhead(gp_overhead_table_size{1, 1, 1, 1, 1});
    static const char* zones[] = {"z0", "z1", "z2"};
    static const char* groups[] = {"g0", "g1", "g2", "gx", ""};
    static const char* letters = "abz09-.";
    std::map<std::string, Host> live;
    auto event = [&](const std::string& name) {
        Host h;
        if (pick(7) != 0) h.labels[NodeTableLabels::kZoneLabel] = zones[pick(3)];
        if (pick(5) != 0) h.labels["instance-group"] = groups[pick(5)];
        h.alloc = resources::CreateResources(16000 * (1 + pick(3)), (int64_t)(64 << pick(2)) << 30, pick(3));
        h.unschedulable = pick(12) == 0;
        h.ready = pick(12) != 0;
        h.creation = 1000 * (int64_t)pick(40);             // few distinct times: equal creation times are common
        live[name] = h;
        labels.SetNode(Node{name, h.labels});
        nodes.SetNode(name, h.alloc, h.unschedulable, h.ready, h.creation);
    };
    int refusedSteps = 0, placedSeen = 0, fallbacks = 0;
    for (int step = 0; step < 14; ++step) {
        for (int e = 0; e < (step == 0 ? 160 : 25); ++e) {
            const int r = pick(10);
            if (r < 5 || live.size() < 8) {
                std::string name;
                for (int k = 0; k < 1 + pick(5); ++k) name += letters[pick(7)];
                if (!live.count(name)) event(name);
            } else if (r < 7) {
                auto it = std::next(live.begin(), pick((int)live.size()));
                nodes.DeleteNode(it->first);
                labels.DeleteNode(it->first);
                live.erase(it);
            } else {
                event(std::next(live.begin(), pick((int)live.size()))->first);
            }
        }
        std::vector<std::string> names;
        for (const auto& kv : live) if (pick(8) != 0 || names.empty()) names.push_back(kv.first);
        std::shuffle(names.begin(), names.end(), rng);
        ResidentReservations::Entries res;
        for (int k = 0; k < 20; ++k)
            res["r" + std::to_string(k)] = {names[(size_t)pick((int)names.size())], resources::CreateResources(500 * pick(8), (int64_t)pick(8) << 30, 0)};
        reservations.SetSoftReservations("app" + std::to_string(step % 3), res);
        labels.Flush(dev);
        nodes.Flush(dev);
        if (step == 9) {                                    // the device's node table replaced behind the host's back
            gp_node_table_size tiny{1, 0};
            dev.check(gp_node_table_reset(dev.ctx(), &tiny), "gp_node_table_reset");
        }

        // the reconciler: every value listed on steps 0, 3, ..; "gx" left out on the others.  On steps 1, 4, .. some driver
        // names "gx", which puts it among the call's groups; on steps 2, 5, .. none does, and the device call is refused
        // whenever a listed node carries "gx" (the host path then replays and answers from the resident path)
        const bool short_list = step % 3 != 0, gx_driver = step % 3 == 1;
        std::vector<std::string> listed = {"g0", "g1", "g2"};
        if (!short_list) listed.push_back("gx");
        std::vector<extender::StaleDriver> drivers;
        for (int i = 0; i < 24; ++i) {
            extender::StaleDriver d;
            d.InstanceGroup = i % 7 == 6 ? "gy" : groups[pick(5)];          // "gy": no node has it
            if (d.InstanceGroup == "gx" && !gx_driver && short_list) d.InstanceGroup = "g0";
            if (i == 0 && gx_driver) d.InstanceGroup = "gx";
            d.ExecutorResources = resources::CreateResources(1000 * (1 + pick(12)), (int64_t)(1 + pick(24)) << 30, pick(4) == 0);
            d.MinExecutorCount = pick(6);
            d.RunningExecutors = pick(3);
            drivers.push_back(d);
        }
        bool carriesGx = false;
        std::vector<ReconcileNode> rn;
        for (const auto& nm : names) {
            const Host& h = live[nm];
            ReconcileNode n;
            n.Name = nm; n.Allocatable = h.alloc; n.Unschedulable = h.unschedulable; n.Ready = h.ready; n.CreationUnixNano = h.creation;
            n.Labels.insert(h.labels.begin(), h.labels.end());
            auto g = h.labels.find("instance-group");
            carriesGx |= g != h.labels.end() && g->second == "gx";
            rn.push_back(n);
        }
        const int replays = nodes.Replays();
        const std::vector<ReconcileResult> a =
            extender::ReconcileFindNodesNodeTable(names, nodes, labels, reservations, overhead, "instance-group", listed, drivers);
        // the device call answered unless it had to refuse: "gx" carried and in no group of the call, or the table reset
        const bool refuse = (short_list && !gx_driver && carriesGx) || step == 9;
        EXPECT((nodes.Replays() != replays) == refuse);
        fallbacks += refuse;
        const std::vector<ReconcileResult> b = extender::ReconcileFindNodesResident(rn, reservations, overhead, "instance-group", drivers);
        EXPECT(same(a, b));
        for (const auto& r : a) placedSeen += (int)r.ReservedNodeNames.size();

        // the raw entry on the tables as they are now: refused exactly when a listed node carries an unlisted value
        {
            std::vector<std::string> g = listed;
            g.push_back("");
            const NodeTableLabels ig(labels, {}, "instance-group", g);
            const std::vector<int32_t> tid = nodes.NodeIDs(names), rid = reservations.NodeIDs(names), oid = overhead.NodeIDs(names);
            gp_node_table_nodes nd{};
            ig.Fill(&nd);
            nd.zone_key = -1; nd.n_zones = 1; nd.zone_value = nullptr; nd.zone_missing = -1;
            nd.n_nodes = (int32_t)names.size(); nd.node_table_id = tid.data(); nd.reservation_id = rid.data(); nd.overhead_node_id = oid.data();
            gp_apps none{};
            std::vector<int64_t> avail(names.size() + 1);
            gp_reconcile_results out{};
            out.avail_cpu_milli = avail.data();
            const gp_status st = gp_reconcile_find_nodes_node_table(dev.ctx(), &nd, (int32_t)g.size(), (int32_t)g.size() - 1, &none, &out);
            EXPECT(st == (short_list && carriesGx ? GP_ERR_INVALID : GP_OK));
            refusedSteps += st != GP_OK;
        }

        // the marker, by node class and by required affinity
        const UnschedulablePodMarker marker(*binpacker::SelectBinpacker(step % 2 ? binpacker::SingleAzTightlyPack : binpacker::tightlyPack));
        std::unordered_map<std::string, int32_t> nodeClass;
        for (const auto& nm : names) if (pick(3) != 0) nodeClass[nm] = pick(2);
        std::vector<UnschedulablePodMarker::StaleDriver> md;
        std::vector<UnschedulablePodMarker::AffinityStaleDriver> ad;
        for (int i = 0; i < 16; ++i) {
            UnschedulablePodMarker::StaleDriver d;
            d.DriverResources = resources::CreateResources(1000 * (1 + pick(8)), (int64_t)(1 + pick(16)) << 30, 0);
            d.ExecutorResources = resources::CreateResources(1000 * (1 + pick(16)), (int64_t)(1 + pick(32)) << 30, 0);
            d.MinExecutorCount = pick(40);
            d.AffinityClass = pick(3) - 1;
            md.push_back(d);
            UnschedulablePodMarker::AffinityStaleDriver x;
            x.DriverResources = d.DriverResources; x.ExecutorResources = d.ExecutorResources; x.MinExecutorCount = d.MinExecutorCount;
            x.Affinity = pick(3);
            ad.push_back(x);
        }
        std::vector<UnschedulablePodMarker::CapacityNode> cn;
        for (const auto& nm : names) {
            UnschedulablePodMarker::CapacityNode c;
            c.Name = nm; c.Allocatable = live[nm].alloc;
            auto z = live[nm].labels.find(NodeTableLabels::kZoneLabel);
            if (z != live[nm].labels.end()) c.ZoneLabel = z->second;
            cn.push_back(c);
        }
        const std::vector<std::string> zl = {"z0", "z1", "z2"};
        const int markerReplays = nodes.Replays();
        EXPECT(marker.DoesPodsExceedClusterCapacity(names, nodes, labels, overhead, zl, nodeClass, 2, md) ==
               marker.DoesPodsExceedClusterCapacity(cn, overhead, nodeClass, 2, md));
        std::vector<Program> programs(3);
        programs[0].NodeSelector["instance-group"] = "g0";
        programs[1].NodeSelector[NodeTableLabels::kZoneLabel] = "z1";
        std::vector<bool> errA, errB;
        EXPECT(marker.DoesPodsExceedClusterCapacity(names, nodes, labels, overhead, zl, programs, ad, &errA) ==
               marker.DoesPodsExceedClusterCapacity(cn, overhead, labels, programs, ad, &errB));
        EXPECT(errA == errB);
        EXPECT(nodes.Replays() == markerReplays);           // both sweeps answered on the device
    }
    EXPECT(refusedSteps > 0);
    EXPECT(fallbacks > 1);                                   // the table reset, and at least one step with "gx" carried
    EXPECT(placedSeen > 0);
    if (failures) { std::printf("host_node_table_reconcile_test: %d failures\n", failures); return 1; }
    std::printf("host_node_table_reconcile_test: all passed\n");
    return 0;
}
