// extender::OverheadComputer (one gp_node_overhead call per query) driven by pod informer events, against a literal
// restatement of overhead.go over the same events: map[node]map[UID] records, a lister lookup, PodHasReservation.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using extender::Container;
using extender::OverheadView;
using extender::Pod;
using resources::Resources;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

namespace literal {
struct Info { std::string name, ns; Resources req; };
struct Computer {
    std::map<std::string, std::map<std::string, Info>> requests;
    void add(const Pod& p) { requests[p.NodeName][p.UID] = Info{p.Name, p.Namespace, extender::PodToResources(p)}; }
    void del(const Pod& p) {
        auto& m = requests[p.NodeName];
        if (!m.count(p.UID)) return;
        m.erase(p.UID);
        if (m.empty()) requests.erase(p.NodeName);
    }
    void onAdd(const Pod& p) { if (!p.NodeName.empty()) add(p); }
    void onUpdate(const Pod& o, const Pod& n) {
        if (!n.NodeName.empty() && o.NodeName.empty()) add(n);
        else if (n.NodeName.empty() && !o.NodeName.empty()) del(o);
    }
    void onDelete(const Pod& p) { if (!p.NodeName.empty()) del(p); }
};
bool hasReservation(const Pod& pod, const OverheadView& v) {
    auto app = pod.Labels.find("spark-app-id");
    if (app == pod.Labels.end()) return false;
    auto rr = v.ResourceReservations.find({pod.Namespace, app->second});
    if (rr != v.ResourceReservations.end())
        for (const auto& n : rr->second) if (n == pod.Name) return true;
    auto role = pod.Labels.find("spark-role");
    if (role != pod.Labels.end() && role->second == "executor") {
        auto sr = v.SoftReservations.find(app->second);
        if (sr != v.SoftReservations.end())
            for (const auto& n : sr->second) if (n == pod.Name) return true;
    }
    return false;
}
void overhead(const Computer& c, const OverheadView& v, const std::string& node, Resources* ov, Resources* ns, int64_t* warned) {
    *ov = Resources{}; *ns = Resources{};
    auto it = c.requests.find(node);
    if (it == c.requests.end()) return;
    for (const auto& kv : it->second) {
        auto p = v.Pods.find({kv.second.ns, kv.second.name});
        if (p == v.Pods.end()) continue;
        const Pod& pod = p->second;
        if (hasReservation(pod, v)) continue;
        ov->Add(kv.second.req);
        if (pod.SchedulerName == "spark-scheduler") {
            auto app = pod.Labels.find("spark-app-id");
            if (v.ResourceReservations.count({pod.Namespace, app == pod.Labels.end() ? std::string() : app->second})) ++*warned;
        } else {
            ns->Add(kv.second.req);
        }
    }
}
}  // namespace literal

static bool Same(const Resources& a, const Resources& b) { return a.CPU == b.CPU && a.Memory == b.Memory && a.NvidiaGPU == b.NvidiaGPU; }

static Pod MakePod(std::mt19937_64& rng, int k, int nNodes) {
    Pod p;
    p.UID = "u" + std::to_string(k);
    p.Namespace = "ns" + std::to_string(rng() % 3);
    p.Name = "p" + std::to_string(rng() % 400);
    p.NodeName = "n" + std::to_string(rng() % (nNodes + 2));
    p.SchedulerName = rng() % 5 < 3 ? "spark-scheduler" : "default-scheduler";
    if (rng() % 5) p.Labels["spark-app-id"] = "app" + std::to_string(rng() % 6);
    if (rng() % 4) p.Labels["spark-role"] = rng() % 3 ? "executor" : "driver";
    p.Containers.push_back(Container{resources::CreateResources((int64_t)(rng() % 4000), (int64_t)(rng() % (1ull << 34)), (int64_t)(rng() % 3))});
    if (rng() % 3 == 0) p.InitContainers.push_back(Container{resources::CreateResources((int64_t)(rng() % 3000), (int64_t)(rng() % (1ull << 33)), 1)});
    return p;
}

int main() {
    {   // podToResources: the per-dimension max with the init containers
        Pod p;
        p.Containers = {Container{resources::CreateResources(100, 10, 0)}, Container{resources::CreateResources(50, 20, 1)}};
        p.InitContainers = {Container{resources::CreateResources(300, 5, 0)}, Container{resources::CreateResources(100, 64, 2)}};
        const Resources r = extender::PodToResources(p);
        EXPECT(r.CPU == 300 && r.Memory == 64 && r.NvidiaGPU == 2);
    }
    for (int seed = 0; seed < 30; ++seed) {
        std::mt19937_64 rng(seed);
        const int nNodes = 1 + seed % 6, nPods = 20 + 40 * seed;
        extender::OverheadComputer comp;
        literal::Computer lit;
        OverheadView v;
        std::vector<Pod> pods;
        for (int k = 0; k < nPods; ++k) {
            Pod p = MakePod(rng, k, nNodes);
            pods.push_back(p);
            if (rng() % 5 == 0) {                              // created unbound, then bound: the update is an add
                Pod unbound = p;
                unbound.NodeName.clear();
                comp.AddPod(unbound); lit.onAdd(unbound);
                comp.UpdatePod(unbound, p); lit.onUpdate(unbound, p);
            } else {
                comp.AddPod(p); lit.onAdd(p);
            }
            if (rng() % 8 == 0) {                              // a later update of a bound pod changes nothing
                Pod resized = p;
                resized.Containers[0].Requests.CPU += 777;
                comp.UpdatePod(p, resized); lit.onUpdate(p, resized);
            }
            if (rng() % 10 == 0) { comp.DeletePod(p); lit.onDelete(p); }
            if (rng() % 10 != 0) v.Pods[{p.Namespace, p.Name}] = p;   // the rest are absent from the lister
        }
        for (int a = 0; a < 6; ++a) {
            const std::string app = "app" + std::to_string(a);
            if (rng() % 3) {
                auto& rr = v.ResourceReservations[{"ns" + std::to_string(rng() % 3), app}];
                for (int j = 0, m = (int)(rng() % 30); j < m; ++j) rr.push_back(pods[rng() % pods.size()].Name);
            }
            if (rng() % 2) {
                auto& sr = v.SoftReservations[app];
                for (int j = 0, m = (int)(rng() % 30); j < m; ++j) sr.push_back(pods[rng() % pods.size()].Name);
            }
        }
        std::vector<std::string> nodes;
        for (int i = nNodes - 1; i >= 0; --i) nodes.push_back("n" + std::to_string(i));
        int64_t warned = -1;
        const auto got = comp.compute(v, nodes, &warned);
        const auto ov = comp.GetOverhead(v, nodes);
        const auto ns = comp.GetNonSchedulableOverhead(v, nodes);
        int64_t want_warned = 0;
        for (const auto& n : nodes) {
            Resources o, s;
            literal::overhead(lit, v, n, &o, &s, &want_warned);
            EXPECT(Same(got.first.at(n), o) && Same(got.second.at(n), s));
            EXPECT(Same(ov.at(n), o) && Same(ns.at(n), s));
        }
        EXPECT(warned == want_warned);
    }
    if (failures) { std::printf("host_overhead_test: %d failures\n", failures); return 1; }
    std::printf("host_overhead_test: all passed\n");
    return 0;
}
