// extender::RescheduleExecutor (one gp_reschedule_from_reservations call) against the string-keyed literal chain of the CPU
// oracle: orc_node_scheduling_metadata + orc_reschedule_available (the two availabilities), orc_potential_nodes (the
// executor order) and orc_reschedule_executor (first fit / minimal fragmentation), after a literal filterNodesToZone when the
// application has a common zone.  Both branches, label priorities, hosting sets, zones that drop out.  Needs an H100.
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "gangpack_host.hpp"
#include "gangpack_oracle.h"   // the CPU oracle is the checker here (tests/ may link it; the product never does)

static int failures = 0;
#define EXPECT(cond, msg)                                                                     \
    do {                                                                                      \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

static const int64_t Gi = 1ll << 30;

static std::vector<const char*> cstrs(const std::vector<std::string>& v) {
    std::vector<const char*> o;
    for (const auto& s : v) o.push_back(s.c_str());
    return o;
}

// the literal chain for one executor over `nodes` (already filtered to the common zone)
static std::string Literal(bool minFrag, const resources::Resources& exe, const std::vector<extender::RescheduleNode>& nodes,
                           const std::vector<extender::ReservationRow>& rows, const resources::NodeGroupResources& overhead,
                           const sort::LabelPriorityOrder* label, const std::set<std::string>& hosting) {
    const size_t n = nodes.size();
    if (n == 0) return "";
    std::vector<std::string> names, zones, rnames;
    std::vector<int64_t> ac, am, ag, oc, om, og, rc, rm, rg;
    std::vector<uint8_t> unsched, ready;
    std::vector<int32_t> lrank;
    for (const auto& nd : nodes) {
        auto beta = nd.AllLabels.find(extender::LabelZoneFailureDomain);             // NodeSchedulingMetadataForNodes :78-81
        names.push_back(nd.Name); zones.push_back(beta == nd.AllLabels.end() ? "default" : beta->second);
        ac.push_back(nd.Allocatable.CPU); am.push_back(nd.Allocatable.Memory); ag.push_back(nd.Allocatable.NvidiaGPU);
        auto o = overhead.find(nd.Name);
        resources::Resources ov = o == overhead.end() ? resources::Resources{} : o->second;
        oc.push_back(ov.CPU); om.push_back(ov.Memory); og.push_back(ov.NvidiaGPU);
        unsched.push_back(nd.Unschedulable); ready.push_back(nd.Ready);
        int32_t r = -1;
        if (label) {
            auto v = nd.AllLabels.find(label->Name);
            for (size_t k = 0; v != nd.AllLabels.end() && k < label->DescendingPriorityValues.size(); ++k)
                if (label->DescendingPriorityValues[k] == v->second) { r = (int32_t)k; break; }
        }
        lrank.push_back(r);
    }
    for (const auto& r : rows) { rnames.push_back(r.Node); rc.push_back(r.Resources.CPU); rm.push_back(r.Resources.Memory); rg.push_back(r.Resources.NvidiaGPU); }
    auto cn = cstrs(names), cz = cstrs(zones), crn = cstrs(rnames);
    std::vector<int64_t> mc(n), mm(n), mg(n), fc(n), fm(n), fg(n);
    orc_node_scheduling_metadata((int32_t)n, cn.data(), ac.data(), am.data(), ag.data(), oc.data(), om.data(), og.data(), (int64_t)rows.size(),
                                 crn.data(), rc.data(), rm.data(), rg.data(), mc.data(), mm.data(), mg.data(), nullptr, nullptr, nullptr);
    orc_reschedule_available((int32_t)n, cn.data(), ac.data(), am.data(), ag.data(), oc.data(), om.data(), og.data(), (int64_t)rows.size(),
                             crn.data(), rc.data(), rm.data(), rg.data(), fc.data(), fm.data(), fg.data());
    orc_cluster* meta = orc_cluster_new((int32_t)n, cn.data(), mc.data(), mm.data(), mg.data(), nullptr, nullptr, nullptr, cz.data(),
                                        unsched.data(), ready.data());
    std::vector<int32_t> drv(n), ex(n);
    int32_t nd = 0, ne = 0;
    orc_potential_nodes(meta, nullptr, 0, nullptr, label ? lrank.data() : nullptr, drv.data(), &nd, ex.data(), &ne);
    std::vector<const char*> order;
    for (int32_t k = 0; k < ne; ++k) order.push_back(cn[(size_t)ex[(size_t)k]]);
    std::vector<std::string> hv(hosting.begin(), hosting.end());
    auto ch = cstrs(hv);
    std::vector<orc_res> res;
    for (size_t i = 0; i < n; ++i) res.push_back(orc_res{oc[i], om[i], og[i]});
    orc_res e{exe.CPU, exe.Memory, exe.NvidiaGPU};
    int32_t w = -1;
    if (minFrag) {
        w = orc_reschedule_executor(meta, 1, &e, order.data(), ne, cn.data(), res.data(), (int32_t)n, ch.data(), (int32_t)ch.size());
    } else {
        orc_cluster* ff = orc_cluster_new((int32_t)n, cn.data(), fc.data(), fm.data(), fg.data(), nullptr, nullptr, nullptr, cz.data(),
                                          unsched.data(), ready.data());
        w = orc_reschedule_executor(ff, 0, &e, order.data(), ne, nullptr, nullptr, 0, nullptr, 0);
        orc_cluster_free(ff);
    }
    orc_cluster_free(meta);
    return w >= 0 ? names[(size_t)w] : "";
}

int main() {
    std::mt19937_64 rng(20261015);
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    const binpacker::Binpacker& ff = binpacker::binpackFunctions().at(binpacker::tightlyPack);
    const binpacker::Binpacker& mf = binpacker::binpackFunctions().at(binpacker::SingleAzMinimalFragmentation);
    sort::LabelPriorityOrder label{"instance-group", {"gold", "silver"}};
    const char* values[] = {"gold", "silver", "bronze"};
    int decisions = 0, found = 0, scoped = 0;
    for (int trial = 0; trial < 40; ++trial) {
        const int n = (int)U(1, 400), zones = (int)U(1, 5);
        std::vector<extender::RescheduleNode> nodes;
        resources::NodeGroupResources overhead;
        for (int i = 0; i < n; ++i) {
            extender::RescheduleNode nd;
            char buf[16]; std::snprintf(buf, sizeof buf, "n%05d", (int)((i * 7919) % 100000));
            nd.Name = buf;
            nd.Allocatable = resources::CreateResources(U(2, 64) * 1000 + U(0, 9) * 7, U(4, 256) * Gi + U(0, 9) * 4096, 0);
            const std::string topo = "z" + std::to_string(U(0, zones - 1));
            nd.AllLabels[extender::LabelTopologyZone] = topo;
            switch (U(0, 2)) {      // the sorter's beta label: absent ("default"), the same zone, or another one (App. B5)
                case 0: break;
                case 1: nd.AllLabels[extender::LabelZoneFailureDomain] = topo; break;
                default: nd.AllLabels[extender::LabelZoneFailureDomain] = "b" + std::to_string(U(0, zones)); break;
            }
            nd.Unschedulable = U(0, 9) == 0; nd.Ready = U(0, 19) != 0;
            if (U(0, 3)) nd.AllLabels["instance-group"] = values[U(0, 2)];
            overhead[nd.Name] = resources::CreateResources(U(0, 2) * 250, U(0, 3) * (Gi / 4), 0);
            nodes.push_back(nd);
        }
        std::vector<extender::ReservationRow> rows;
        for (int r = 0, R = (int)U(0, 3 * n); r < R; ++r)
            rows.push_back({U(0, 20) ? nodes[(size_t)U(0, n - 1)].Name : std::string("gone"),
                            resources::CreateResources(U(0, 8) * 500, U(0, 16) * (Gi / 2), 0)});
        for (int x = 0; x < 12; ++x) {
            const bool useMf = x & 1, useLabel = (x >> 1) & 1;
            const resources::Resources exe = resources::CreateResources(U(0, 8) * 500, U(0, 32) * (Gi / 2), 0);
            std::set<std::string> hosting;
            for (int h = 0, H = (int)U(0, 4); h < H; ++h) hosting.insert(nodes[(size_t)U(0, n - 1)].Name);
            std::string zone;
            const std::string* common = nullptr;
            if (x >= 6) { zone = "z" + std::to_string(U(0, zones)); common = &zone; ++scoped; }     // z<zones>: no node kept
            std::vector<extender::RescheduleNode> kept;
            for (const auto& nd : nodes)                                                             // filterNodesToZone
                if (!common || nd.AllLabels.at(extender::LabelTopologyZone) == zone) kept.push_back(nd);
            auto got = extender::RescheduleExecutor(useMf ? mf : ff, exe, nodes, rows, overhead, useLabel ? &label : nullptr, common, hosting);
            const std::string want = Literal(useMf, exe, kept, rows, overhead, useLabel ? &label : nullptr, hosting);
            EXPECT(got.Node == want && got.Found == !want.empty(), (std::string("trial ") + std::to_string(trial) + " exec " + std::to_string(x) +
                                                                   " got " + got.Node + " want " + want).c_str());
            EXPECT(!got.Ambiguous, "no gpu column: never ambiguous");
            ++decisions; found += got.Found;
        }
    }
    // the sorter zone is the beta label, not the topology label: without the beta label every node is in zone "default", so
    // the emptier zone z1 does not come first.  a: 8 cores / 8 GiB in z1; b, c: 6 / 6 in z2 -> the reference chooses b.
    {
        std::vector<extender::RescheduleNode> nodes(3);
        const char* nm[] = {"a", "b", "c"};
        const int64_t size[] = {8, 6, 6};
        const char* topo[] = {"z1", "z2", "z2"};
        for (int i = 0; i < 3; ++i) {
            nodes[i].Name = nm[i];
            nodes[i].Allocatable = resources::CreateResources(size[i] * 1000, size[i] * Gi, 0);
            nodes[i].AllLabels[extender::LabelTopologyZone] = topo[i];
        }
        auto got = extender::RescheduleExecutor(ff, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, nullptr, {});
        EXPECT(got.Found && got.Node == "b", ("beta label missing: got " + got.Node).c_str());
        EXPECT(Literal(false, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, {}) == "b", "literal chooses b");
        for (int i = 0; i < 3; ++i) nodes[i].AllLabels[extender::LabelZoneFailureDomain] = topo[i];    // now the zones count
        got = extender::RescheduleExecutor(ff, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, nullptr, {});
        EXPECT(got.Found && got.Node == "a", ("beta label = topology label: got " + got.Node).c_str());
        const std::string z2 = "z2";                 // scope by the topology label while the beta labels say otherwise
        for (int i = 0; i < 3; ++i) nodes[i].AllLabels[extender::LabelZoneFailureDomain] = "elsewhere";
        got = extender::RescheduleExecutor(ff, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, &z2, {});
        EXPECT(got.Found && got.Node == "b", ("scope z2: got " + got.Node).c_str());
    }
    // a node without the topology label fails the scoped call, like filterNodesToZone
    {
        std::vector<extender::RescheduleNode> nodes(3);
        for (int i = 0; i < 3; ++i) {
            nodes[i].Name = "m" + std::to_string(i); nodes[i].Allocatable = resources::CreateResources(4000, 8 * Gi, 0);
            nodes[i].AllLabels[extender::LabelTopologyZone] = "z0"; nodes[i].AllLabels[extender::LabelZoneFailureDomain] = "z0";
        }
        nodes[2].AllLabels.erase(extender::LabelTopologyZone);
        const std::string zone = "z0";
        bool threw = false;
        try {
            extender::RescheduleExecutor(ff, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, &zone, {});
        } catch (const gangpack::Error& e) {
            threw = std::string(e.what()).find("filterNodesToZone") != std::string::npos;
        }
        EXPECT(threw, "missing zone label must be refused");
        auto any = extender::RescheduleExecutor(ff, resources::CreateResources(1000, Gi, 0), nodes, {}, {}, nullptr, nullptr, {});
        EXPECT(any.Found, "without a scope the label is not read");
    }
    EXPECT(found > 50 && found < decisions && scoped > 100, "coverage");
    std::printf("%d decisions, %d found, %d scoped\n", decisions, found, scoped);
    if (failures) { std::printf("%d failures\n", failures); return 1; }
    std::printf("all passed\n");
    return 0;
}
