// extender::ResidentOverheadComputer (one gp_overhead_table_update and one gp_overhead_table_query per compute) driven by
// pod, lister, ResourceReservation and soft-store events, against a literal restatement of overhead.go over the same
// events -- map[node]map[UID] records, a lister lookup, PodHasReservation by scanning Status.Pods -- and against
// extender::OverheadComputer (gp_node_overhead) on the same views.
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
    p.Name = "p" + std::to_string(rng() % 80);
    p.NodeName = "n" + std::to_string(rng() % (nNodes + 2));
    p.SchedulerName = rng() % 5 < 3 ? "spark-scheduler" : "default-scheduler";
    if (rng() % 5) p.Labels["spark-app-id"] = "app" + std::to_string(rng() % 6);
    if (rng() % 4) p.Labels["spark-role"] = rng() % 3 ? "executor" : "driver";
    p.Containers.push_back(Container{resources::CreateResources((int64_t)(rng() % 4000), (int64_t)(rng() % (1ull << 34)), (int64_t)(rng() % 3))});
    if (rng() % 3 == 0) p.InitContainers.push_back(Container{resources::CreateResources((int64_t)(rng() % 3000), (int64_t)(rng() % (1ull << 33)), 1)});
    return p;
}

int main() {
    int computes = 0;
    for (int seed = 0; seed < 20; ++seed) {
        std::mt19937_64 rng(1000 + seed);
        const int nNodes = 1 + seed % 6;
        extender::ResidentOverheadComputer comp(gp_overhead_table_size{2, 1, 1, 1, 2});   // small: capacities double and replay
        extender::OverheadComputer perCall;
        literal::Computer lit;
        OverheadView v;
        std::map<std::string, Pod> live;                   // uid -> the pod's current object
        std::vector<std::string> nodes;
        for (int i = nNodes - 1; i >= 0; --i) nodes.push_back("n" + std::to_string(i));
        auto names = [&](int m) {
            std::vector<std::string> out;
            for (int j = 0; j < m; ++j) out.push_back("p" + std::to_string(rng() % 82));   // repeats, and names of no pod
            return out;
        };
        int uid = 0;
        for (int step = 0; step < 40; ++step) {
            for (int e = 0, n = 1 + (int)(rng() % 8); e < n; ++e) {
                const int op = (int)(rng() % 12);
                auto pick = [&]() { auto it = live.begin(); std::advance(it, (long)(rng() % live.size())); return it; };
                if (op <= 2 || live.empty()) {                         // a new pod, bound or not, usually listed
                    Pod p = MakePod(rng, uid++, nNodes);
                    if (rng() % 4 == 0) p.NodeName.clear();
                    comp.AddPod(p); perCall.AddPod(p); lit.onAdd(p);
                    live[p.UID] = p;
                    if (rng() % 5) { v.Pods[{p.Namespace, p.Name}] = p; comp.SetListerPod(p); }
                } else if (op == 3) {                                  // bind, or update a bound pod (no change)
                    auto it = pick();
                    Pod q = it->second;
                    if (q.NodeName.empty()) q.NodeName = "n" + std::to_string(rng() % (nNodes + 2));
                    else q.Containers[0].Requests.CPU += 777;
                    comp.UpdatePod(it->second, q); perCall.UpdatePod(it->second, q); lit.onUpdate(it->second, q);
                    it->second = q;
                } else if (op == 4) {                                  // unbind
                    auto it = pick();
                    Pod q = it->second;
                    q.NodeName.clear();
                    comp.UpdatePod(it->second, q); perCall.UpdatePod(it->second, q); lit.onUpdate(it->second, q);
                    it->second = q;
                } else if (op == 5) {                                  // delete, usually gone from the lister too
                    auto it = pick();
                    const Pod p = it->second;
                    live.erase(it);
                    comp.DeletePod(p); perCall.DeletePod(p); lit.onDelete(p);
                    if (rng() % 3) { v.Pods.erase({p.Namespace, p.Name}); comp.DeleteListerPod(p.Namespace, p.Name); }
                } else if (op == 6) {                                  // the lister's pod changes labels, role, scheduler
                    auto it = pick();
                    Pod q = MakePod(rng, 0, nNodes);
                    q.Namespace = it->second.Namespace; q.Name = it->second.Name; q.UID = it->second.UID;
                    v.Pods[{q.Namespace, q.Name}] = q;
                    comp.SetListerPod(q);
                } else if (op == 7) {
                    auto it = pick();
                    v.Pods.erase({it->second.Namespace, it->second.Name});
                    comp.DeleteListerPod(it->second.Namespace, it->second.Name);
                } else if (op == 8) {                                  // an RR created or rewritten
                    const std::string ns = "ns" + std::to_string(rng() % 3), app = "app" + std::to_string(rng() % 6);
                    const auto pods = names((int)(rng() % 10));
                    v.ResourceReservations[{ns, app}] = pods;
                    comp.SetResourceReservation(ns, app, pods);
                } else if (op == 9 && !v.ResourceReservations.empty()) {
                    auto it = v.ResourceReservations.begin();
                    std::advance(it, (long)(rng() % v.ResourceReservations.size()));
                    comp.DeleteResourceReservation(it->first.first, it->first.second);
                    v.ResourceReservations.erase(it);
                } else if (op == 10) {
                    const std::string app = "app" + std::to_string(rng() % 6);
                    const auto pods = names((int)(rng() % 8));
                    v.SoftReservations[app] = pods;
                    comp.SetSoftReservation(app, pods);
                } else if (op == 11 && !v.SoftReservations.empty()) {
                    auto it = v.SoftReservations.begin();
                    std::advance(it, (long)(rng() % v.SoftReservations.size()));
                    comp.DeleteSoftReservation(it->first);
                    v.SoftReservations.erase(it);
                }
            }
            int64_t warned = -1, callWarned = -1;
            const auto got = comp.compute(nodes, &warned);
            const auto call = perCall.compute(v, nodes, &callWarned);
            ++computes;
            int64_t want = 0;
            for (const auto& n : nodes) {
                Resources o, s;
                literal::overhead(lit, v, n, &o, &s, &want);
                EXPECT(Same(got.first.at(n), o) && Same(got.second.at(n), s));
                EXPECT(Same(call.first.at(n), o) && Same(call.second.at(n), s));
            }
            EXPECT(warned == want && callWarned == want);
        }
        const auto ov = comp.GetOverhead(nodes);                      // nothing changed: no update, one query
        const auto ns = comp.GetNonSchedulableOverhead(nodes);
        int64_t want = 0;
        for (const auto& n : nodes) {
            Resources o, s;
            literal::overhead(lit, v, n, &o, &s, &want);
            EXPECT(Same(ov.at(n), o) && Same(ns.at(n), s));
        }
    }
    if (failures) { std::printf("host_resident_overhead_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_overhead_test: all passed (%d computes)\n", computes);
    return 0;
}
