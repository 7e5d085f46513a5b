// resources::ResidentNodes and resources::NodeTableLabels (the C++ host layer of the resident node table) driven by random
// node add / update / delete events with capacities that double from one and 10-bit name keys (frequent relabels), next to
// affinity::ResidentLabels, extender::ResidentReservations and an extender::ResidentOverheadComputer.  After every flush,
// gp_prepare_cluster_groups_node_table and gp_reschedule_from_reservations_node_table must equal the *_resident entries given
// the host's per-call columns (ResidentNodes::PerCall, NodeTableLabels::Decode of the label strings, names sorted on the
// host) -- counts, orders, offsets, ties, the snapshot and the node choice.  A node table replaced behind the host's back
// (a reset) makes the next call refuse; Replay and Flush restore it.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using affinity::Node;
using affinity::ResidentLabels;
using extender::ResidentOverheadComputer;
using extender::ResidentReservations;
using resources::NodeTableLabels;
using resources::ResidentNodes;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

struct Outcome {
    gp_status st = GP_OK;
    int32_t nd = 0, ne = 0, ties = 0;
    std::vector<int32_t> eoff, drvoff, eorder, dorder, igTies;
    std::vector<int64_t> snap[3];
    bool operator==(const Outcome& o) const {
        return st == o.st && nd == o.nd && ne == o.ne && ties == o.ties && eoff == o.eoff && drvoff == o.drvoff && eorder == o.eorder &&
               dorder == o.dorder && igTies == o.igTies && snap[0] == o.snap[0] && snap[1] == o.snap[1] && snap[2] == o.snap[2];
    }
};

// runs one prepare call into fresh output buffers, then reads the snapshot back
template <class F>
static Outcome run(gangpack::Device& dev, size_t n, int32_t G, int32_t* ties, F&& call) {
    Outcome o;
    o.eoff.assign(G + 1, -9); o.drvoff.assign(G + 1, -9); o.eorder.assign(n, -9); o.dorder.assign(n, -9); o.igTies.assign(G, -9);
    gp_instance_group_orders out{0, 0, o.eoff.data(), o.eorder.data(), o.drvoff.data(), o.dorder.data(), o.igTies.data()};
    *ties = -9;
    o.st = call(&out);
    if (o.st != GP_OK) { Outcome refused; refused.st = o.st; return refused; }
    o.nd = out.n_driver; o.ne = out.n_executor; o.ties = *ties;
    for (auto& v : o.snap) v.assign(n, 0);
    dev.check(gp_get_snapshot(dev.ctx(), o.snap[0].data(), o.snap[1].data(), o.snap[2].data()), "gp_get_snapshot");
    return o;
}

int main() {
    std::mt19937_64 rng(77);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    gangpack::Device& dev = gangpack::Device::Get();
    ResidentLabels labels(gp_label_table_size{1, 1, 1, 1});
    ResidentNodes nodes(labels, 1, 10);
    ResidentReservations reservations(gp_reservation_table_size{1, 1});
    ResidentOverheadComputer overhead(gp_overhead_table_size{1, 1, 1, 1, 1});
    const sort::LabelPriorityOrder drvPrio{"priority", {"p1", "p0", "p2", "p1"}}, exePrio{"priority", {"p2", "p0"}};
    static const char* zones[] = {"z0", "z1", "z2"};
    static const char* groups[] = {"g0", "g1", "g2", "gx"};
    static const char* prio[] = {"p0", "p1", "p2", "px"};
    static const char* letters = "abz09-.";
    std::map<std::string, std::map<std::string, std::string>> live;
    auto event = [&](const std::string& name) {
        std::map<std::string, std::string> l;
        if (pick(7) != 0) l[NodeTableLabels::kZoneLabel] = zones[pick(3)];
        if (pick(5) != 0) l["instance-group"] = groups[pick(4)];
        if (pick(2) != 0) l["priority"] = prio[pick(4)];
        live[name] = l;
        labels.SetNode(Node{name, l});
        nodes.SetNode(name, resources::CreateResources(16000 * (1 + pick(3)), (int64_t)(64 << pick(2)) << 30, pick(3)), pick(20) == 0,
                      pick(20) != 0);
    };
    int64_t tiesSeen = 0;
    for (int step = 0; step < 16; ++step) {
        for (int e = 0; e < (step == 0 ? 200 : 30); ++e) {
            const int r = pick(10);
            if (r < 5 || live.size() < 8) {
                std::string name;
                if (pick(3) == 0 && !live.empty()) name = std::next(live.begin(), pick((int)live.size()))->first + letters[pick(7)];
                else for (int k = 0; k < 1 + pick(5); ++k) name += letters[pick(7)];
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
        reservations.Flush(dev);
        overhead.Flush(dev);
        if (step == 9) {                                    // the device's node table replaced behind the host's back
            gp_node_table_size tiny{1, 0};
            dev.check(gp_node_table_reset(dev.ctx(), &tiny), "gp_node_table_reset");
        }

        const size_t n = names.size();
        const NodeTableLabels cfg(labels, {"z0", "z1", "z2"}, "instance-group", {"g0", "g1", "g2"}, step % 2 ? &drvPrio : nullptr,
                                  step % 2 ? &exePrio : nullptr);
        const std::vector<int32_t> tid = nodes.NodeIDs(names), rid = reservations.NodeIDs(names), oid = overhead.NodeIDs(names);
        std::vector<uint8_t> cand(n);
        for (auto& c : cand) c = pick(10) != 0;
        int32_t tiesA = 0, tiesB = 0;
        gp_node_table_nodes nt{};
        nt.n_nodes = (int32_t)n; nt.node_table_id = tid.data(); nt.reservation_id = rid.data(); nt.overhead_node_id = oid.data();
        nt.is_driver_candidate = cand.data(); nt.undefined_ties = &tiesA;
        cfg.Fill(&nt);
        const int32_t G = cfg.NumInstanceGroups();
        Outcome a = run(dev, n, G, &tiesA, [&](gp_instance_group_orders* out) {
            return gp_prepare_cluster_groups_node_table(dev.ctx(), &nt, nullptr, G, out);
        });
        if (step == 9) {
            EXPECT(a.st == GP_ERR_INVALID);
            nodes.Replay();
            nodes.Flush(dev);
            a = run(dev, n, G, &tiesA, [&](gp_instance_group_orders* out) {
                return gp_prepare_cluster_groups_node_table(dev.ctx(), &nt, nullptr, G, out);
            });
        }
        // the *_resident form over the host's columns
        const ResidentNodes::Columns col = nodes.PerCall(names);
        std::vector<Node> nds;
        for (const auto& nm : names) nds.push_back(Node{nm, live[nm]});
        NodeTableLabels::Columns lab;
        EXPECT(cfg.Decode(nds, &lab));
        gp_resident_usage ru{(int32_t)n, rid.data(), col.alloc[0].data(), col.alloc[1].data(), col.alloc[2].data(), oid.data(), nullptr, nullptr,
                             nullptr};
        gp_sort_input si{};
        si.n_nodes = (int32_t)n; si.n_zones = cfg.NumZones(); si.zone_id = lab.zone.data(); si.name_rank = col.nameRank.data();
        si.is_driver_candidate = cand.data(); si.unschedulable = col.unschedulable.data(); si.ready = col.ready.data();
        si.driver_label_rank = lab.driverRank.empty() ? nullptr : lab.driverRank.data();
        si.executor_label_rank = lab.executorRank.empty() ? nullptr : lab.executorRank.data();
        si.undefined_ties = &tiesB;
        const Outcome b = run(dev, n, G, &tiesB, [&](gp_instance_group_orders* out) {
            return gp_prepare_cluster_groups_resident(dev.ctx(), &ru, &si, lab.instanceGroup.data(), G, out);
        });
        EXPECT(a.st == GP_OK);
        EXPECT(a == b);
        tiesSeen += b.ties;

        // the executor Predicate: first fit and minimal fragmentation
        const int32_t q = 12;
        std::vector<int64_t> ec(q), em(q), eg(q);
        for (int32_t i = 0; i < q; ++i) { ec[i] = 1000 * (1 + pick(20)); em[i] = (int64_t)(1 + pick(64)) << 30; eg[i] = pick(3) == 0; }
        for (int mf = 0; mf < 2; ++mf) {
            gp_reschedule rq{};
            rq.n_execs = q; rq.exe_cpu_milli = ec.data(); rq.exe_mem_bytes = em.data(); rq.exe_gpu = eg.data(); rq.min_frag = mf;
            std::vector<int32_t> outA(q, -9), outB(q, -9);
            std::vector<uint8_t> ambA(q, 9), ambB(q, 9);
            EXPECT(gp_reschedule_from_reservations_node_table(dev.ctx(), &nt, nullptr, &rq, outA.data(), ambA.data()) == GP_OK);
            EXPECT(gp_reschedule_from_reservations_resident(dev.ctx(), &ru, &si, nullptr, &rq, outB.data(), ambB.data()) == GP_OK);
            EXPECT(outA == outB && ambA == ambB);
        }
    }
    EXPECT(nodes.Relabels() > 0);
    EXPECT(tiesSeen > 0);
    if (failures) { std::printf("host_resident_nodes_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_nodes_test: all passed\n");
    return 0;
}
