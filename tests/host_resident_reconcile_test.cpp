// extender::ReconcileFindNodesResident and UnschedulablePodMarker's resident sweep (each table's pending delta flushed once,
// then one gp_reconcile_find_nodes_resident / gp_exceeds_cluster_capacity_resident call) driven by random ResourceReservation,
// soft-store and pod events, against the per-call host entries on a literal restatement of the same state: every reservation
// row from the test's own maps, the overhead from ResidentOverheadComputer's query.  Includes a refused reservation update
// (a value >= 2^61) followed by the replay that brings the table back.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using extender::ResidentOverheadComputer;
using extender::ResidentReservations;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

static bool same(const std::vector<extender::ReconcileResult>& a, const std::vector<extender::ReconcileResult>& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if (a[i].InstanceGroupFound != b[i].InstanceGroupFound || a[i].ReservedNodeNames != b[i].ReservedNodeNames) return false;
    return true;
}

int main() {
    std::mt19937_64 rng(29);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    std::vector<std::string> names;
    for (int i = 0; i < 24; ++i) names.push_back("node-" + std::to_string(i));
    ResidentReservations table(gp_reservation_table_size{1, 1});
    ResidentOverheadComputer overhead(gp_overhead_table_size{1, 1, 1, 1, 1});
    std::map<std::string, ResidentReservations::Entries> rrs, soft;          // the restatement's own view of the events
    auto entries = [&](const std::string& prefix) {
        ResidentReservations::Entries e;
        const int k = pick(5);
        for (int j = 0; j < k; ++j) {
            resources::Resources r;
            r.CPU = pick(8) * 500; r.Memory = (int64_t)pick(16) << 28; r.NvidiaGPU = pick(3) == 0;
            const std::string node = pick(8) == 0 ? "gone-" + std::to_string(pick(2)) : names[(size_t)pick((int)names.size())];
            e[prefix + std::to_string(j)] = ResidentReservations::Reservation{node, r};
        }
        return e;
    };
    std::vector<extender::ReconcileNode> nodes;
    std::vector<extender::UnschedulablePodMarker::CapacityNode> cap;
    for (size_t i = 0; i < names.size(); ++i) {
        extender::ReconcileNode n;
        n.Name = names[i];
        n.Allocatable = resources::CreateResources(8000 + pick(8) * 1000, (int64_t)(16 + pick(48)) << 30, pick(3));
        n.Labels["ig"] = "ig-" + std::to_string(pick(3));
        n.Unschedulable = pick(10) == 0; n.Ready = pick(10) != 0;
        n.CreationUnixNano = pick(20);
        nodes.push_back(n);
        cap.push_back({names[i], n.Allocatable, "zone-" + std::to_string(pick(2))});
    }
    std::unordered_map<std::string, int32_t> nodeClass;
    for (const auto& n : names) if (pick(4) != 0) nodeClass[n] = pick(2);
    int uid = 0, checked = 0;
    for (int step = 0; step < 40; ++step) {
        for (int ev = 0; ev < 1 + pick(6); ++ev) {
            const std::string app = "app-" + std::to_string(pick(10));
            switch (pick(5)) {
            case 0: { auto e = entries(app + "-e"); table.SetResourceReservation("ns", app, e); if (e.empty()) rrs.erase(app); else rrs[app] = e; break; }
            case 1: table.DeleteResourceReservation("ns", app); rrs.erase(app); break;
            case 2: { auto e = entries(app + "-p" + std::to_string(step)); table.SetSoftReservations(app, e); if (e.empty()) soft.erase(app); else soft[app] = e; break; }
            case 3: table.DeleteSoftReservations(app); soft.erase(app); break;
            default: {                                   // a pod without a reservation: overhead on its node
                extender::Pod p;
                p.UID = "u" + std::to_string(uid); p.Namespace = "ns"; p.Name = "pod-" + std::to_string(uid++);
                p.NodeName = names[(size_t)pick((int)names.size())];
                p.SchedulerName = pick(2) ? "spark-scheduler" : "default-scheduler";
                p.Containers.push_back({resources::CreateResources(pick(4) * 250, (int64_t)pick(4) << 28, 0)});
                overhead.AddPod(p);
                overhead.SetListerPod(p);
                break;
            }
            }
        }
        std::vector<extender::StaleDriver> drivers;
        std::vector<extender::UnschedulablePodMarker::StaleDriver> stale;
        for (int i = 0; i < 1 + pick(12); ++i) {
            extender::StaleDriver d;
            d.InstanceGroup = "ig-" + std::to_string(pick(4));                      // ig-3 has no node
            d.ExecutorResources = resources::CreateResources(500 * (1 + pick(8)), (int64_t)(1 + pick(8)) << 30, pick(5) == 0);
            d.MinExecutorCount = pick(6); d.RunningExecutors = pick(3);
            drivers.push_back(d);
            extender::UnschedulablePodMarker::StaleDriver s;
            s.DriverResources = resources::CreateResources(1000, 2ll << 30, 0);
            s.ExecutorResources = d.ExecutorResources;
            s.MinExecutorCount = pick(40);
            s.AffinityClass = pick(3) - 1;
            stale.push_back(s);
        }
        if (step == 20) {                                // a refused update: the table replays once the value is fixed
            ResidentReservations::Entries bad{{"x", {names[0], resources::CreateResources(int64_t(1) << 61, 0, 0)}}};
            table.SetResourceReservation("ns", "bad", bad);
            bool refused = false;
            try { extender::ReconcileFindNodesResident(nodes, table, overhead, "ig", drivers); }
            catch (const gangpack::Error& e) { refused = e.status == GP_ERR_UNREPRESENTABLE; }
            EXPECT(refused);
            table.DeleteResourceReservation("ns", "bad");
        }
        std::vector<extender::ReconcileRow> rows;
        for (const auto* store : {&rrs, &soft})
            for (const auto& owner : *store)
                for (const auto& e : owner.second) rows.push_back({e.second.Node, e.second.Res});
        const auto got = extender::ReconcileFindNodesResident(nodes, table, overhead, "ig", drivers);
        const auto want = extender::ReconcileFindNodes(nodes, rows, overhead.GetOverhead(names), "ig", drivers);
        EXPECT(same(got, want));
        const binpacker::Binpacker packer = *binpacker::SelectBinpacker(step % 2 ? binpacker::SingleAzTightlyPack : binpacker::tightlyPack);
        const extender::UnschedulablePodMarker marker(packer);
        const auto gotEx = marker.DoesPodsExceedClusterCapacity(cap, overhead, nodeClass, 2, stale);
        const resources::NodeGroupResources nonsched = overhead.GetNonSchedulableOverhead(names);
        resources::NodeGroupSchedulingMetadata md;
        for (const auto& c : cap) {
            resources::NodeSchedulingMetadata m;
            m.SchedulableResources = c.Allocatable;
            m.SchedulableResources.Sub(nonsched.at(c.Name));
            m.ZoneLabel = c.ZoneLabel;
            md[c.Name] = m;
        }
        EXPECT(gotEx == marker.DoesPodsExceedClusterCapacity(md, nodeClass, 2, stale));
        ++checked;
    }
    if (failures) { std::printf("host_resident_reconcile_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_reconcile_test: all passed (%d reconciles)\n", checked);
    return 0;
}
