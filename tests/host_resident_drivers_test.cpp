// extender::ResidentDrivers and extender::FitEarlierDriversDriverTable (the C++ host layer of the resident driver table)
// driven by random pending-driver pod events -- adds, updates, bound and terminating pods, unparseable annotations -- with
// capacities that double from one.  After every batch of events the table form must equal the per-call recipe on the
// same pods, computed here independently: FilterToEarliestAndSort over the listed pods, PendingDriverFromAnnotations,
// shouldSkipDriverFifo, then FitEarlierDrivers for the earlier drivers and for the requesting one -- the status, the
// requesting driver's packing result, the undefined ties and the metadata left behind.  A driver table replaced behind the
// host's back by one without slots makes the next flush or call refuse; the call replays the table and answers from the
// per-call path, and the call after it is answered by the table again.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "gangpack_host.hpp"

using extender::DriverQueueOutcome;
using extender::QueuedDriverPod;
using extender::ResidentDrivers;
using resources::NodeGroupSchedulingMetadata;

static int failures = 0;
#define EXPECT(c)                                                                  \
    do {                                                                           \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++failures; } \
    } while (0)

static const int64_t kSec = 1000000000LL;

struct Pod {
    QueuedDriverPod pod;
    std::map<std::string, std::string> annotations;
};

// the per-call recipe over the host's own copy of the pods
// (listed in slot order: the order in which the table breaks equal creation times, which the reference's unstable sort.Slice
// leaves undefined -- undefinedTies counts them)
static DriverQueueOutcome PerCall(const binpacker::Binpacker& packer, const std::map<std::string, Pod>& pods, const ResidentDrivers& table,
                                  const std::string& uid, const std::map<std::string, int64_t>& ages, int64_t defaultAge, int64_t now,
                                  const std::vector<std::string>& names, NodeGroupSchedulingMetadata& md) {
    std::vector<QueuedDriverPod> listed;
    for (const auto& kv : pods) listed.push_back(kv.second.pod);
    std::sort(listed.begin(), listed.end(), [&](const QueuedDriverPod& x, const QueuedDriverPod& y) { return table.Slot(x.UID) < table.Slot(y.UID); });
    DriverQueueOutcome out;
    const QueuedDriverPod& me = pods.at(uid).pod;
    std::vector<extender::PendingDriver> queue;
    auto earlier = extender::FilterToEarliestAndSort(me, listed);
    for (size_t j = 0; j < earlier.size(); ++j) {
        const auto& p = earlier[j];
        auto a = ages.find(p.InstanceGroup);
        const int64_t age = a == ages.end() ? defaultAge : a->second;
        queue.push_back(extender::PendingDriverFromAnnotations(p.UID, pods.at(p.UID).annotations, p.CreationSeconds * kSec + age > now));
        if (j > 0 && p.CreationSeconds == earlier[j - 1].CreationSeconds) ++out.undefinedTies;
    }
    if (!extender::FitEarlierDrivers(packer, queue, names, names, md)) { out.status = -2; return out; }
    std::vector<binpack::PackingResult> res;
    extender::FitEarlierDrivers(packer, {extender::PendingDriverFromAnnotations(uid, pods.at(uid).annotations, false)}, names, names, md, &res);
    out.result = res[0];
    out.status = res[0].HasCapacity ? 0 : -1;
    return out;
}

int main() {
    std::mt19937_64 rng(91);
    auto pick = [&](int n) { return (int)(rng() % (uint64_t)n); };
    gangpack::Device& dev = gangpack::Device::Get();
    std::vector<std::string> names;
    NodeGroupSchedulingMetadata base;
    for (int i = 0; i < 24; ++i) {
        names.push_back("node-" + std::to_string(i));
        resources::NodeSchedulingMetadata m;
        m.AvailableResources = resources::CreateResources(1000 * (2 + pick(6)), (int64_t)(4 + pick(12)) << 30, pick(2));
        m.SchedulableResources = m.AvailableResources;
        base[names.back()] = m;
    }
    const char* groups[] = {"g0", "g1", "g2"};
    const std::map<std::string, int64_t> ages{{"g1", 120 * kSec}, {"g2", -5 * kSec}};
    const int64_t defaultAge = 30 * kSec, now = 1000 * kSec;
    ResidentDrivers drivers(gp_driver_table_size{1, 1, 1, 0});
    std::map<std::string, Pod> pods;             // the pending, parseable drivers
    int next = 0, fromTable = 0, fellBack = 0, compared = 0;
    for (int step = 0; step < 40; ++step) {
        for (int e = 0; e < 1 + pick(12); ++e) {
            Pod p;
            const bool update = !pods.empty() && pick(3) == 0;
            p.pod.UID = update ? std::next(pods.begin(), pick((int)pods.size()))->first : "driver-" + std::to_string(next++);
            p.pod.CreationSeconds = 900 + pick(100);
            p.pod.SchedulerName = pick(8) == 0 ? "other" : "spark-scheduler";
            p.pod.HasInstanceGroup = pick(10) != 0;
            if (p.pod.HasInstanceGroup) p.pod.InstanceGroup = groups[pick(3)];
            p.annotations = {{"spark-driver-cpu", std::to_string(1 + pick(3))}, {"spark-driver-mem", std::to_string(1 + pick(3)) + "Gi"},
                             {"spark-executor-cpu", std::to_string(1 + pick(3))}, {"spark-executor-mem", std::to_string(1 + pick(4)) + "Gi"},
                             {"spark-executor-count", std::to_string(pick(5))}};
            const int kind = pick(20);
            if (kind == 0) p.pod.NodeName = "node-0";                      // bound
            else if (kind == 1) p.pod.Deleting = true;                     // terminating
            else if (kind == 2) p.annotations["spark-driver-cpu"] = "x";   // unparseable
            drivers.SetDriver(p.pod, p.annotations);
            if (kind <= 2) pods.erase(p.pod.UID);
            else pods[p.pod.UID] = p;
        }
        if (pods.empty()) continue;
        if (step % 7 == 3) {                      // the device's table replaced by one without slots behind the host's back
            gp_driver_table_size z = drivers.Size();
            z.n_slots = 0;
            dev.check(gp_driver_table_reset(dev.ctx(), &z), "gp_driver_table_reset");
        }
        for (int k = 0; k < 3; ++k) {
            const std::string uid = std::next(pods.begin(), pick((int)pods.size()))->first;
            for (const char* pk : {"tightly-pack", "distribute-evenly"}) {
                const binpacker::Binpacker& packer = *binpacker::SelectBinpacker(pk);
                NodeGroupSchedulingMetadata a = base, b = base;
                const int replays = drivers.Replays();
                const DriverQueueOutcome got = extender::FitEarlierDriversDriverTable(packer, drivers, uid, defaultAge, ages, now, names, names, a);
                const DriverQueueOutcome want = PerCall(packer, pods, drivers, uid, ages, defaultAge, now, names, b);
                EXPECT((got.status >= 0) == (want.status >= 0) && (got.status < 0 ? got.status == want.status : true));
                EXPECT(got.result.HasCapacity == want.result.HasCapacity && got.result.DriverNode == want.result.DriverNode &&
                       got.result.ExecutorNodes == want.result.ExecutorNodes);
                EXPECT(got.undefinedTies == want.undefinedTies);
                for (const auto& n : names) {
                    const auto& x = a.at(n).AvailableResources;
                    const auto& y = b.at(n).AvailableResources;
                    EXPECT(x.CPU == y.CPU && x.Memory == y.Memory && x.NvidiaGPU == y.NvidiaGPU);
                }
                if (got.fromTable) ++fromTable;
                else { ++fellBack; EXPECT(drivers.Replays() == replays + 1); }
                ++compared;
            }
        }
    }
    EXPECT(fromTable > 0 && fellBack > 0);
    // the zone-aware packers are answered by the per-call path
    {
        const std::string uid = pods.begin()->first;
        NodeGroupSchedulingMetadata a = base;
        EXPECT(!extender::FitEarlierDriversDriverTable(*binpacker::SelectBinpacker("single-az-tightly-pack"), drivers, uid, defaultAge, ages, now,
                                                       names, names, a).fromTable);
    }
    std::printf("compared %d calls: %d from the table, %d after a refusal\n", compared, fromTable, fellBack);
    if (failures) { std::printf("host_resident_drivers_test: %d failures\n", failures); return 1; }
    std::printf("host_resident_drivers_test: all passed\n");
    return 0;
}
