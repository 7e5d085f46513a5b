// extender::ReconcileFindNodes (one gp_reconcile_find_nodes call per reconciliation) against the string-keyed C literal of
// availableResourcesPerInstanceGroup + findNodes + the charge loop (tests/reconcile_oracle.c).  Random clusters with nodes and
// drivers that have no instance-group label (the "" group), drivers of groups without nodes, unschedulable and not-ready nodes,
// creation ties, reservation rows on nodes outside the table, soft rows and running executors.  Needs an H100.
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "gangpack_host.hpp"

extern "C" int orc_reconcile_find_nodes(int32_t n, const char** names, const int64_t* alloc_cpu, const int64_t* alloc_mem,
                                        const int64_t* alloc_gpu, const char** group_label, const uint8_t* unschedulable,
                                        const uint8_t* ready, const int64_t* creation, const int64_t* over_cpu, const int64_t* over_mem,
                                        const int64_t* over_gpu, int64_t n_rows, const char** row_node, const int64_t* row_cpu,
                                        const int64_t* row_mem, const int64_t* row_gpu, int32_t q, const char** drv_group,
                                        const int64_t* exe_cpu, const int64_t* exe_mem, const int64_t* exe_gpu, const int32_t* min_count,
                                        const int32_t* running, int32_t* placed, int32_t* out_nodes, int64_t* avail_cpu,
                                        int64_t* avail_mem, int64_t* avail_gpu);

static int failures = 0;
#define EXPECT(cond, msg)                                                            \
    do {                                                                             \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

static const int64_t Gi = 1ll << 30;
static const char* kLabel = "resource_channel";

static void Trial(std::mt19937_64& rng, int n, int nGroups, int q, int nRows) {
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    std::vector<extender::ReconcileNode> nodes(n);
    resources::NodeGroupResources overhead;
    for (int i = 0; i < n; ++i) {
        auto& nd = nodes[i];
        nd.Name = "node-" + std::to_string(i);
        nd.Allocatable = resources::CreateResources(U(0, 32) * 1000, U(0, 128) * Gi, U(0, 3) == 0 ? U(0, 8) : 0);
        const int64_t g = U(0, nGroups);                                     // nGroups: no label at all
        if (g < nGroups) nd.Labels[kLabel] = g == 0 ? "" : "ig-" + std::to_string(g);
        nd.Labels["other"] = "x";
        nd.Unschedulable = U(0, 9) == 0;
        nd.Ready = U(0, 9) != 0;
        nd.CreationUnixNano = U(0, n / 3 + 1) * 1000000000ll;
        if (U(0, 1)) overhead[nd.Name] = resources::CreateResources(U(0, 1500), U(0, 2) * Gi, 0);
    }
    std::vector<extender::ReconcileRow> rows(nRows);
    for (auto& r : rows) {
        const int64_t v = U(-1, n - 1);
        r.Node = v < 0 ? "gone-" + std::to_string(U(0, 99)) : nodes[v].Name;
        r.Resources = resources::CreateResources(U(0, 8) * 1000, U(0, 32) * Gi, U(0, 1));
    }
    std::vector<extender::StaleDriver> drivers(q);
    for (auto& d : drivers) {
        const int64_t g = U(0, nGroups + 1);                                 // nGroups + 1: a group no node carries
        d.InstanceGroup = g == 0 || g == nGroups ? "" : "ig-" + std::to_string(g);
        const int64_t shape = U(0, 4);
        d.ExecutorResources = resources::CreateResources(shape == 0 ? 0 : U(1, 6) * 500, shape == 1 ? 0 : U(1, 16) * Gi, shape == 2 ? 1 : 0);
        if (shape == 3) d.ExecutorResources = resources::Zero();
        d.MinExecutorCount = (int)U(0, 30);
        d.RunningExecutors = U(0, 3) == 0 ? (int)U(0, 40) : 0;
    }
    const auto got = extender::ReconcileFindNodes(nodes, rows, overhead, kLabel, drivers);
    // the literal, string-keyed
    std::vector<const char*> names(n), labels(n), rnode(nRows), dgroup(q);
    std::vector<int64_t> ac(n), am(n), ag(n), oc(n), om(n), og(n), cr(n), rc(nRows), rm(nRows), rg(nRows), ec(q), em(q), eg(q);
    std::vector<uint8_t> fu(n), fr(n);
    std::vector<int32_t> mn(q), run(q), placed(q + 1);
    int64_t total = 0;
    for (int i = 0; i < n; ++i) {
        names[i] = nodes[i].Name.c_str();
        auto l = nodes[i].Labels.find(kLabel);
        labels[i] = l == nodes[i].Labels.end() ? nullptr : l->second.c_str();
        ac[i] = nodes[i].Allocatable.CPU; am[i] = nodes[i].Allocatable.Memory; ag[i] = nodes[i].Allocatable.NvidiaGPU;
        auto o = overhead.find(nodes[i].Name);
        if (o != overhead.end()) { oc[i] = o->second.CPU; om[i] = o->second.Memory; og[i] = o->second.NvidiaGPU; }
        fu[i] = nodes[i].Unschedulable; fr[i] = nodes[i].Ready; cr[i] = nodes[i].CreationUnixNano;
    }
    for (int r = 0; r < nRows; ++r) {
        rnode[r] = rows[r].Node.c_str();
        rc[r] = rows[r].Resources.CPU; rm[r] = rows[r].Resources.Memory; rg[r] = rows[r].Resources.NvidiaGPU;
    }
    for (int i = 0; i < q; ++i) {
        dgroup[i] = drivers[i].InstanceGroup.c_str();
        ec[i] = drivers[i].ExecutorResources.CPU; em[i] = drivers[i].ExecutorResources.Memory; eg[i] = drivers[i].ExecutorResources.NvidiaGPU;
        mn[i] = drivers[i].MinExecutorCount; run[i] = drivers[i].RunningExecutors;
        total += std::max(0, mn[i] - std::min(run[i], mn[i]));
    }
    std::vector<int32_t> out(total + 1);
    std::vector<int64_t> av(3 * (size_t)(n + 1));
    const int bad = orc_reconcile_find_nodes(n, names.data(), ac.data(), am.data(), ag.data(), labels.data(), fu.data(), fr.data(), cr.data(),
                                             oc.data(), om.data(), og.data(), nRows, rnode.data(), rc.data(), rm.data(), rg.data(), q,
                                             dgroup.data(), ec.data(), em.data(), eg.data(), mn.data(), run.data(), placed.data(), out.data(),
                                             av.data(), av.data() + n + 1, av.data() + 2 * (n + 1));
    EXPECT(!bad, "the literal left the exact domain");
    EXPECT(got.size() == (size_t)q, "one result per driver");
    int64_t off = 0;
    for (int i = 0; i < q && i < (int)got.size(); ++i) {
        EXPECT(got[i].InstanceGroupFound == (placed[i] >= 0), "instance group found");
        if (placed[i] >= 0) {
            EXPECT(got[i].ReservedNodeNames.size() == (size_t)placed[i], "len(reservedNodeNames)");
            for (int j = 0; j < placed[i] && j < (int)got[i].ReservedNodeNames.size(); ++j)
                EXPECT(got[i].ReservedNodeNames[j] == nodes[out[off + j]].Name, "reservedNodeNames");
        }
        off += std::max(0, mn[i] - std::min(run[i], mn[i]));
    }
}

int main() {
    std::mt19937_64 rng(20261016);
    for (int t = 0; t < 300; ++t) Trial(rng, 1 + (int)(rng() % 200), 1 + (int)(rng() % 6), (int)(rng() % 60), (int)(rng() % 400));
    Trial(rng, 5000, 12, 2000, 20000);
    if (failures) { std::printf("%d failures\n", failures); return 1; }
    std::printf("all passed\n");
    return 0;
}
