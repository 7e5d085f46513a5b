// extender::ResidentReservations (at most one gp_reservation_table_update per Predicate, then
// gp_prepare_cluster_groups_resident) driven by random ResourceReservation and soft-store events -- creates, rewrites,
// deletes, capacities that double from 1 -- against a literal restatement of GetReservedResources over the same events:
// map[name]Reservation per ResourceReservation and per soft-store application, summed per node name.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using extender::ResidentReservations;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

// UsageForNodes + UsedSoftReservationResources, string-keyed
static std::map<std::string, resources::Resources> reserved(const std::map<std::string, ResidentReservations::Entries>& rrs,
                                                            const std::map<std::string, ResidentReservations::Entries>& soft) {
    std::map<std::string, resources::Resources> u;
    for (const auto* store : {&rrs, &soft})
        for (const auto& owner : *store)
            for (const auto& e : owner.second) {
                auto& r = u[e.second.Node];
                r.CPU += e.second.Res.CPU; r.Memory += e.second.Res.Memory; r.NvidiaGPU += e.second.Res.NvidiaGPU;
            }
    return u;
}

int main() {
    gangpack::Device& dev = gangpack::Device::Get();
    std::mt19937_64 rng(17);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    std::vector<std::string> names;
    for (int i = 0; i < 12; ++i) names.push_back("node-" + std::to_string(i));
    ResidentReservations table(gp_reservation_table_size{1, 1});
    std::map<std::string, ResidentReservations::Entries> rrs, soft;          // the restatement's own view of the events
    auto entries = [&](const std::string& prefix) {
        ResidentReservations::Entries e;
        const int k = pick(5);
        for (int j = 0; j < k; ++j) {
            resources::Resources r;
            r.CPU = pick(8) * 500 - (pick(10) == 0 ? 7 : 0); r.Memory = (int64_t)pick(16) << 28; r.NvidiaGPU = pick(3);
            e[prefix + std::to_string(j)] = ResidentReservations::Reservation{names[(size_t)pick((int)names.size())], r};
        }
        return e;
    };
    const int64_t alloc = int64_t(1) << 50;
    int checked = 0;
    for (int step = 0; step < 60; ++step) {
        for (int ev = 0; ev < 1 + pick(6); ++ev) {
            const std::string app = "app-" + std::to_string(pick(10));
            switch (pick(4)) {
            case 0: { auto e = entries(app + "-e"); table.SetResourceReservation("ns", app, e); if (e.empty()) rrs.erase(app); else rrs[app] = e; break; }
            case 1: table.DeleteResourceReservation("ns", app); rrs.erase(app); break;
            case 2: { auto e = entries(app + "-p" + std::to_string(step)); table.SetSoftReservations(app, e); if (e.empty()) soft.erase(app); else soft[app] = e; break; }
            default: table.DeleteSoftReservations(app); soft.erase(app); break;
            }
        }
        table.Flush(dev);
        // the Predicate's node table: a shuffled subset (nodes outside it keep their reservations, which are not counted)
        std::vector<std::string> nodes;
        for (const auto& n : names) if (pick(5) != 0) nodes.push_back(n);
        std::shuffle(nodes.begin(), nodes.end(), rng);
        if (nodes.empty()) continue;
        const int32_t n = (int32_t)nodes.size();
        const std::vector<int32_t> ids = table.NodeIDs(nodes);
        std::vector<int64_t> a(nodes.size(), alloc);
        gp_resident_usage u{n, ids.data(), a.data(), a.data(), nullptr, nullptr, nullptr, nullptr, nullptr};
        gp_sort_input s{};
        s.n_nodes = n; s.n_zones = 1;
        gp_instance_group_orders o{};
        dev.check(gp_prepare_cluster_groups_resident(dev.ctx(), &u, &s, nullptr, 1, &o), "gp_prepare_cluster_groups_resident");
        std::vector<int64_t> cpu(nodes.size()), mem(nodes.size()), gpu(nodes.size());
        dev.check(gp_get_snapshot(dev.ctx(), cpu.data(), mem.data(), gpu.data()), "gp_get_snapshot");
        const auto want = reserved(rrs, soft);
        for (size_t i = 0; i < nodes.size(); ++i) {
            auto it = want.find(nodes[i]);
            const resources::Resources w = it == want.end() ? resources::Resources{} : it->second;
            EXPECT(alloc - cpu[i] == w.CPU && alloc - mem[i] == w.Memory && -gpu[i] == w.NvidiaGPU);
        }
        ++checked;
    }
    EXPECT(checked > 40);
    if (failures) { std::printf("host_resident_reservations_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_reservations_test: all passed (%d Predicates)\n", checked);
    return 0;
}
