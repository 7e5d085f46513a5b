// UnschedulablePodMarker's driver-table scan (the C++ host layer of gp_exceeds_cluster_capacity_driver_table) against the
// per-call node-table affinity sweep on the same pods, driven by random node and pending-driver pod events: adds, updates,
// bound and terminating pods, unparseable annotations, other schedulers and a few distinct required affinities (one of
// which errors on every node).  The per-call side is computed here independently: the stale filter over the test's own pods,
// (creation, slot) order, the affinities listed by the test and one that matches every node.  A stale driver's affinity id
// rewritten out of range behind the host's back makes the call refuse; the scan replays the tables and answers per call,
// and the scan after it is answered by the table again.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using affinity::Node;
using affinity::Program;
using affinity::ResidentLabels;
using extender::ParsedSparkResources;
using extender::QueuedDriverPod;
using extender::ResidentDrivers;
using extender::ResidentOverheadComputer;
using extender::UnschedulablePodMarker;
using resources::NodeTableLabels;
using resources::ResidentNodes;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

static const int64_t kSec = 1000000000LL;

struct Pod {
    QueuedDriverPod pod;
    std::map<std::string, std::string> annotations;
    int affinity = -1;                     // index into the test's programs, -1: none
};

int main() {
    std::mt19937_64 rng(17);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    gangpack::Device& dev = gangpack::Device::Get();
    ResidentLabels labels(gp_label_table_size{1, 1, 1, 1});
    ResidentNodes nodes(labels, 1, 10);
    ResidentOverheadComputer overhead(gp_overhead_table_size{1, 1, 1, 1, 1});
    ResidentDrivers drivers(gp_driver_table_size{1, 1, 1, 0});
    static const char* zones[] = {"z0", "z1", "z2"};
    static const char* groups[] = {"g0", "g1", "g2"};
    std::vector<std::string> names;
    for (int i = 0; i < 40; ++i) {
        names.push_back("n" + std::to_string(i));
        std::map<std::string, std::string> lab{{NodeTableLabels::kZoneLabel, zones[pick(3)]}};
        if (pick(5) != 0) lab["instance-group"] = groups[pick(3)];
        labels.SetNode(Node{names.back(), lab});
        nodes.SetNode(names.back(), resources::CreateResources(16000 * (1 + pick(3)), (int64_t)(64 << pick(2)) << 30, pick(3)), false, true);
    }
    std::vector<Program> programs(3);
    programs[0].NodeSelector["instance-group"] = "g0";
    programs[1].NodeSelector[NodeTableLabels::kZoneLabel] = "z1";
    programs[2].HasRequired = true;                         // Gt with a value that is not an integer: an error on every node
    programs[2].Terms.push_back(affinity::Term{{affinity::Requirement{"instance-group", "Gt", {"x"}}}, {}});
    const std::vector<std::string> zl = {"z0", "z1", "z2"};
    const int64_t timeout = 50 * kSec, now = 1000 * kSec;
    std::map<std::string, Pod> pods;                        // the pending, parseable drivers
    int next = 0, fromTable = 0, fellBack = 0, scanned = 0, errors = 0;
    for (int step = 0; step < 24; ++step) {
        for (int e = 0; e < (step == 0 ? 150 : 1 + pick(20)); ++e) {
            Pod p;
            const bool update = !pods.empty() && pick(3) == 0;
            p.pod.UID = update ? std::next(pods.begin(), pick((int)pods.size()))->first : "driver-" + std::to_string(next++);
            p.pod.CreationSeconds = 900 + pick(100);
            p.pod.SchedulerName = pick(8) == 0 ? "other" : "spark-scheduler";
            p.pod.HasInstanceGroup = pick(10) != 0;
            if (p.pod.HasInstanceGroup) p.pod.InstanceGroup = groups[pick(3)];
            p.affinity = pick(5) - 2 < 0 ? -1 : pick(3);
            if (p.affinity >= 0) p.pod.Affinity = programs[(size_t)p.affinity];
            p.annotations = {{"spark-driver-cpu", std::to_string(1 + pick(3))}, {"spark-driver-mem", std::to_string(1 + pick(3)) + "Gi"},
                             {"spark-executor-cpu", std::to_string(1 + pick(8))}, {"spark-executor-mem", std::to_string(1 + pick(16)) + "Gi"},
                             {"spark-executor-count", std::to_string(pick(30))}};
            const int kind = pick(20);
            if (kind == 0) p.pod.NodeName = "n0";                          // bound
            else if (kind == 1) p.pod.Deleting = true;                     // terminating
            else if (kind == 2) p.annotations["spark-driver-cpu"] = "x";   // unparseable
            drivers.SetDriver(p.pod, p.annotations);
            if (kind <= 2) pods.erase(p.pod.UID);
            else pods[p.pod.UID] = p;
        }
        // the per-call recipe over the test's own pods (flushed first, so that the slots are the table's)
        drivers.Flush(dev);
        std::vector<const Pod*> stale;
        for (const auto& kv : pods)
            if (kv.second.pod.SchedulerName == "spark-scheduler" && kv.second.pod.CreationSeconds * kSec + timeout < now) stale.push_back(&kv.second);
        std::sort(stale.begin(), stale.end(), [&](const Pod* a, const Pod* b) {
            return a->pod.CreationSeconds != b->pod.CreationSeconds ? a->pod.CreationSeconds < b->pod.CreationSeconds
                                                                    : drivers.Slot(a->pod.UID) < drivers.Slot(b->pod.UID);
        });
        std::vector<Program> progs = programs;
        progs.push_back(Program{});
        std::vector<UnschedulablePodMarker::AffinityStaleDriver> ad;
        for (const Pod* p : stale) {
            ParsedSparkResources r;
            extender::SparkResources(p->annotations, &r);
            UnschedulablePodMarker::AffinityStaleDriver d;
            d.DriverResources = resources::CreateResources(r.DriverCPUMilli, r.DriverMemoryBytes, r.DriverNvidiaGPUs);
            d.ExecutorResources = resources::CreateResources(r.ExecutorCPUMilli, r.ExecutorMemoryBytes, r.ExecutorNvidiaGPUs);
            d.MinExecutorCount = (int)r.MinExecutorCount;
            d.Affinity = p->affinity < 0 ? (int)programs.size() : p->affinity;
            ad.push_back(d);
        }
        const UnschedulablePodMarker marker(*binpacker::SelectBinpacker(step % 2 ? binpacker::SingleAzTightlyPack : binpacker::tightlyPack));
        std::vector<bool> err;
        const std::vector<bool> exceeds = marker.DoesPodsExceedClusterCapacity(names, nodes, labels, overhead, zl, progs, ad, &err);
        const bool force = step % 6 == 4 && !stale.empty();
        if (force) {                                        // a stale driver's affinity id out of range, behind the host's back
            const Pod& p = *stale[0];
            ParsedSparkResources r;
            extender::SparkResources(p.annotations, &r);
            const int32_t slot = drivers.Slot(p.pod.UID), sched = drivers.SchedulerID("spark-scheduler"), grp = -1,
                          count = (int32_t)r.MinExecutorCount, aff = 999;
            const uint8_t on = 1, exact = 1;
            const int64_t cre = p.pod.CreationSeconds * kSec;
            gp_driver_delta d{1, 0, &slot, &on, &cre, &sched, &grp, &r.DriverCPUMilli, &r.DriverMemoryBytes, &r.DriverNvidiaGPUs,
                              &r.ExecutorCPUMilli, &r.ExecutorMemoryBytes, &r.ExecutorNvidiaGPUs, &count, &exact, &aff};
            dev.check(gp_driver_table_update(dev.ctx(), &d), "gp_driver_table_update");
        }
        const int replays = drivers.Replays();
        const auto got = marker.DoesPodsExceedClusterCapacity(drivers, "spark-scheduler", timeout, now, names, nodes, labels, overhead, zl);
        EXPECT(marker.LastScanFellBack() == force);
        EXPECT(drivers.Replays() == replays + (force ? 1 : 0));
        EXPECT(got.size() == stale.size());
        for (size_t i = 0; i < std::min(got.size(), stale.size()); ++i) {
            EXPECT(got[i].UID == stale[i]->pod.UID);
            EXPECT(got[i].Outcome == (err[i] ? 1 : 0));
            EXPECT(got[i].Exceeds == exceeds[i]);
            errors += got[i].Outcome == 1;
        }
        (force ? fellBack : fromTable) += 1;
        scanned += (int)got.size();
        for (int k = 0; k < 4 && !pods.empty(); ++k) {       // bound or deleted since the scan
            const std::string uid = std::next(pods.begin(), pick((int)pods.size()))->first;
            drivers.DeleteDriver(uid);
            pods.erase(uid);
        }
    }
    EXPECT(fromTable > 0 && fellBack > 0 && errors > 0);
    std::printf("compared %d scans (%d stale drivers): %d from the table, %d after a refusal\n", fromTable + fellBack, scanned, fromTable,
                fellBack);
    if (failures) { std::printf("host_resident_marker_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_marker_test: all passed\n");
    return 0;
}
