// gangpack_host.hpp -- C++ host-side mirror of the reference's plug-in interface for the placement
// hot path, implemented over the C ABI (include/gangpack.h).  The Go toolchain is absent in this
// environment, so this is the host layer a maintainer can compile and test; go/binpacker_gpu.go is
// the same thing as a cgo shim.  Names, argument meaning and error behaviour follow the reference:
//
//   resources::Resources / NodeSchedulingMetadata / NodeGroupSchedulingMetadata
//        vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg/resources/resources.go:103-246
//   binpack::PackingResult / SparkBinPackFunction / TightlyPack / DistributeEvenly
//        vendor/.../pkg/binpack/binpack.go:25-48, pack_tightly.go:25-32, distribute_evenly.go:25-32
//   binpacker::Binpacker / SelectBinpacker        internal/binpacker/binpack.go:37-58
//   sort::NodeSorter::PotentialNodes              internal/sort/nodesorting.go:41-200
//   extender::FitEarlierDrivers / SparkResourceUsage
//        internal/extender/resource.go:224-262, internal/extender/sparkpods.go:139-146
//   extender::ResidentDrivers / FitEarlierDriversDriverTable (pending drivers kept on the device, the FIFO step from them)
//        internal/extender/sparkpods.go:45-137, internal/extender/resource.go:224-270
//
// Quantities are int64 (CPU millicores, memory bytes, GPU units) -- the exact-int64 model of
// resource.Quantity.  There is no CPU packer here: if the device path fails the call throws
// gangpack::Error unless a fallback packer has been installed (the Go shim installs the original
// Go function, see INTEGRATION.md).
#pragma once

#include <algorithm>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "gangpack.h"
#include "spark_resources.hpp"

namespace gangpack {
struct Error : std::runtime_error {
    int status;
    Error(int st, const std::string& m) : std::runtime_error(m), status(st) {}
};
}  // namespace gangpack

// ------------------------------------------------------------------------------------------------
namespace resources {

struct Resources {                       // resources.go:151-155
    int64_t CPU = 0;        // millicores
    int64_t Memory = 0;     // bytes
    int64_t NvidiaGPU = 0;  // units
    bool GreaterThan(const Resources& o) const { return CPU > o.CPU || Memory > o.Memory || NvidiaGPU > o.NvidiaGPU; }  // :239-241
    bool Eq(const Resources& o) const { return CPU == o.CPU && Memory == o.Memory && NvidiaGPU == o.NvidiaGPU; }          // :244-246
    void Add(const Resources& o) { CPU += o.CPU; Memory += o.Memory; NvidiaGPU += o.NvidiaGPU; }                          // :202-206
    void Sub(const Resources& o) { CPU -= o.CPU; Memory -= o.Memory; NvidiaGPU -= o.NvidiaGPU; }                          // :209-213
};
inline Resources Zero() { return Resources{}; }                                                                            // :177-183
inline Resources CreateResources(int64_t cpuMilli, int64_t memory, int64_t gpus) { return Resources{cpuMilli, memory, gpus}; }

struct NodeSchedulingMetadata {          // resources.go:158-166
    Resources AvailableResources;
    Resources SchedulableResources;
    std::string ZoneLabel = "default";   // zoneLabelPlaceholder, :27
    std::map<std::string, std::string> AllLabels;
    bool Unschedulable = false;
    bool Ready = true;
};

using NodeGroupResources = std::unordered_map<std::string, Resources>;                 // :103
struct NodeGroupSchedulingMetadata : std::unordered_map<std::string, NodeSchedulingMetadata> {  // :106
    // SubtractUsageIfExists, :129-135
    void SubtractUsageIfExists(const NodeGroupResources& used) {
        for (const auto& kv : used) {
            auto it = find(kv.first);
            if (it != end()) it->second.AvailableResources.Sub(kv.second);
        }
    }
};

}  // namespace resources

// ------------------------------------------------------------------------------------------------
namespace binpack {

struct PackingResult {                   // binpack.go:25-30 (PackingEfficiencies: metrics by-product, not produced)
    std::string DriverNode;
    std::vector<std::string> ExecutorNodes;
    bool HasCapacity = false;
};
inline PackingResult EmptyPackingResult() { return PackingResult{}; }    // :33-40

using SparkBinPackFunction = std::function<PackingResult(               // :43-48
    const resources::Resources& driverResources, const resources::Resources& executorResources, int executorCount,
    const std::vector<std::string>& driverNodePriorityOrder, const std::vector<std::string>& executorNodePriorityOrder,
    const resources::NodeGroupSchedulingMetadata& nodesSchedulingMetadata)>;

}  // namespace binpack

// ------------------------------------------------------------------------------------------------
namespace gangpack {

// One device context + the marshalling between name-keyed Go-style maps and the SoA buffers.
class Device {
public:
    static Device& Get() {
        static Device d;
        return d;
    }
    gp_ctx* ctx() { return ctx_; }

    // Marshal metadata + the two orders (names absent from the metadata are dropped: they can host
    // neither a driver, binpack.go:68-69, nor an executor, pack_tightly.go:51-52) and upload.
    void SetSnapshot(const resources::NodeGroupSchedulingMetadata& md, const std::vector<std::string>& driverOrder,
                     const std::vector<std::string>& executorOrder) {
        names_.clear(); index_.clear();
        cpu_.clear(); mem_.clear(); gpu_.clear(); exec_.clear(); drv_.clear();
        auto intern = [&](const std::string& n) -> int32_t {
            auto it = index_.find(n);
            if (it != index_.end()) return it->second;
            auto m = md.find(n);
            if (m == md.end()) return -1;
            int32_t i = (int32_t)names_.size();
            names_.push_back(n);
            index_.emplace(n, i);
            cpu_.push_back(m->second.AvailableResources.CPU);
            mem_.push_back(m->second.AvailableResources.Memory);
            gpu_.push_back(m->second.AvailableResources.NvidiaGPU);
            return i;
        };
        std::vector<uint8_t> seen;
        auto add_unique = [&](std::vector<int32_t>& dst, const std::vector<std::string>& src) {
            seen.assign(src.size() + names_.size() + 1, 0);
            for (const auto& n : src) {
                int32_t i = intern(n);
                if (i < 0) continue;
                if ((size_t)i >= seen.size()) seen.resize((size_t)i + 1, 0);
                if (seen[i]) throw Error(GP_ERR_INVALID, "node listed twice in a priority order: " + n);
                seen[i] = 1;
                dst.push_back(i);
            }
        };
        add_unique(exec_, executorOrder);
        add_unique(drv_, driverOrder);
        int32_t eoff[2] = {0, (int32_t)exec_.size()}, doff[2] = {0, (int32_t)drv_.size()};
        gp_nodes n{};
        n.n_nodes = (int32_t)names_.size();
        n.avail_cpu_milli = cpu_.data(); n.avail_mem_bytes = mem_.data(); n.avail_gpu = gpu_.data();
        n.n_groups = 1;
        n.exec_off = eoff; n.exec_order = exec_.data();
        n.drv_off = doff; n.drv_order = drv_.data();
        check(gp_set_snapshot(ctx_, &n), "gp_set_snapshot");
    }
    // One instance group per entry of `groups` (driver order, executor order): used by the single-AZ packers,
    // where a "group" is a zone.  Nodes are interned once; a node may appear in one group only.
    void SetSnapshotGroups(const resources::NodeGroupSchedulingMetadata& md,
                           const std::vector<std::pair<std::vector<std::string>, std::vector<std::string>>>& groups) {
        names_.clear(); index_.clear();
        cpu_.clear(); mem_.clear(); gpu_.clear(); exec_.clear(); drv_.clear();
        std::vector<int32_t> eoff{0}, doff{0};
        auto intern = [&](const std::string& n) -> int32_t {
            auto it = index_.find(n);
            if (it != index_.end()) return it->second;
            auto m = md.find(n);
            if (m == md.end()) return -1;
            int32_t i = (int32_t)names_.size();
            names_.push_back(n);
            index_.emplace(n, i);
            cpu_.push_back(m->second.AvailableResources.CPU);
            mem_.push_back(m->second.AvailableResources.Memory);
            gpu_.push_back(m->second.AvailableResources.NvidiaGPU);
            return i;
        };
        for (const auto& g : groups) {
            for (const auto& n : g.second) { int32_t i = intern(n); if (i >= 0) exec_.push_back(i); }
            for (const auto& n : g.first) { int32_t i = intern(n); if (i >= 0) drv_.push_back(i); }
            eoff.push_back((int32_t)exec_.size());
            doff.push_back((int32_t)drv_.size());
        }
        gp_nodes n{};
        n.n_nodes = (int32_t)names_.size();
        n.avail_cpu_milli = cpu_.data(); n.avail_mem_bytes = mem_.data(); n.avail_gpu = gpu_.data();
        n.n_groups = (int32_t)groups.size();
        n.exec_off = eoff.data(); n.exec_order = exec_.data();
        n.drv_off = doff.data(); n.drv_order = drv_.data();
        check(gp_set_snapshot(ctx_, &n), "gp_set_snapshot");
    }
    // NodeSchedulingMetadata.SchedulableResources of the interned nodes (the packing efficiencies read them)
    void SetSchedulable(const resources::NodeGroupSchedulingMetadata& md) {
        std::vector<int64_t> c(names_.size()), m(names_.size()), g(names_.size());
        for (size_t i = 0; i < names_.size(); ++i) {
            const auto& s = md.at(names_[i]).SchedulableResources;
            c[i] = s.CPU; m[i] = s.Memory; g[i] = s.NvidiaGPU;
        }
        check(gp_set_schedulable(ctx_, c.data(), m.data(), g.data()), "gp_set_schedulable");
    }
    // Every node of the metadata in one executor-only group (no driver candidates): the node table of the
    // cluster-wide packing efficiency (gp_packing_efficiency), with its SchedulableResources
    void SetSnapshotAll(const resources::NodeGroupSchedulingMetadata& md) {
        names_.clear(); index_.clear();
        cpu_.clear(); mem_.clear(); gpu_.clear(); exec_.clear(); drv_.clear();
        for (const auto& kv : md) {
            index_.emplace(kv.first, (int32_t)names_.size());
            exec_.push_back((int32_t)names_.size());
            names_.push_back(kv.first);
            cpu_.push_back(kv.second.AvailableResources.CPU);
            mem_.push_back(kv.second.AvailableResources.Memory);
            gpu_.push_back(kv.second.AvailableResources.NvidiaGPU);
        }
        int32_t eoff[2] = {0, (int32_t)exec_.size()}, doff[2] = {0, 0};
        gp_nodes n{};
        n.n_nodes = (int32_t)names_.size();
        n.avail_cpu_milli = cpu_.data(); n.avail_mem_bytes = mem_.data(); n.avail_gpu = gpu_.data();
        n.n_groups = 1;
        n.exec_off = eoff; n.exec_order = exec_.data();
        n.drv_off = doff; n.drv_order = drv_.data();
        check(gp_set_snapshot(ctx_, &n), "gp_set_snapshot");
        SetSchedulable(md);
    }
    const std::string& name(int32_t i) const { return names_.at((size_t)i); }
    size_t n_nodes() const { return names_.size(); }
    int32_t index(const std::string& n) const { auto it = index_.find(n); return it == index_.end() ? -1 : it->second; }
    void check(int st, const char* what) {
        if (st != GP_OK) throw Error(st, std::string(what) + ": " + gp_last_error(ctx_));
    }

private:
    Device() {
        if (gp_create(&ctx_, nullptr) != GP_OK) throw Error(GP_ERR_NO_DEVICE, std::string("gp_create: ") + gp_last_error(nullptr));
    }
    ~Device() { gp_destroy(ctx_); }
    gp_ctx* ctx_ = nullptr;
    std::vector<std::string> names_;
    std::unordered_map<std::string, int32_t> index_;
    std::vector<int64_t> cpu_, mem_, gpu_;
    std::vector<int32_t> exec_, drv_;
};

// optional CPU fallback installed by the embedding application (the Go shim installs the original packer)
inline std::map<int, binpack::SparkBinPackFunction>& Fallbacks() {
    static std::map<int, binpack::SparkBinPackFunction> f;
    return f;
}

inline binpack::PackingResult PackOne(gp_algo algo, const resources::Resources& drv, const resources::Resources& exe, int count,
                                      const std::vector<std::string>& driverOrder, const std::vector<std::string>& executorOrder,
                                      const resources::NodeGroupSchedulingMetadata& md) {
    try {
        Device& d = Device::Get();
        d.SetSnapshot(md, driverOrder, executorOrder);
        std::vector<int32_t> nodes((size_t)std::max(count, 1));
        int32_t has = 0, driver = -1;
        d.check(gp_pack_one(d.ctx(), algo, drv.CPU, drv.Memory, drv.NvidiaGPU, exe.CPU, exe.Memory, exe.NvidiaGPU, count, &has,
                            &driver, nodes.data()),
                "gp_pack_one");
        binpack::PackingResult r;
        if (!has) return r;                       // EmptyPackingResult
        r.HasCapacity = true;
        r.DriverNode = d.name(driver);
        r.ExecutorNodes.reserve((size_t)count);
        for (int i = 0; i < count; ++i) r.ExecutorNodes.push_back(d.name(nodes[(size_t)i]));
        return r;
    } catch (const Error&) {
        auto f = Fallbacks().find((int)algo);
        if (f != Fallbacks().end() && f->second) return f->second(drv, exe, count, driverOrder, executorOrder, md);
        throw;
    }
}

// What the host side of every resident table (gp_*_table_*) shares: the size the table is reset with, capacities that double
// and force a replay, and the step that sends a delta.  A Flush assembles its delta from the whole state while Replaying(),
// else from what changed, and hands it to Send.
template <class Size>
class ResidentTable {
public:
    // the next Flush resets the table and sends the whole state again (after a refused resident call)
    void Replay() { replay_ = true; ++replays_; }
    int Replays() const { return replays_; }      // Replay calls: a host path's fallback after a refused device call is one

protected:
    explicit ResidentTable(Size initial) : size_(initial) {}
    bool Replaying() const { return replay_; }
    template <class T> void Grow(T& cap, int64_t need) {
        while (cap < need) { cap = std::max<T>(2 * cap, 1); replay_ = true; }
    }
    // The reset when replaying, then the update of *d (none when d is NULL).  Until both calls return the next Flush replays:
    // a call that throws leaves the device's table to be rebuilt.
    template <class Reset, class Update, class Delta>
    void Send(Device& dev, Reset reset, const char* resetName, Update update, const char* updateName, const Delta* d) {
        const bool replaying = replay_;
        replay_ = true;
        if (replaying) dev.check(reset(dev.ctx(), &size_), resetName);
        if (d) dev.check(update(dev.ctx(), d), updateName);
        replay_ = false;
    }

    Size size_;

private:
    bool replay_ = true;
    int replays_ = 0;
};

}  // namespace gangpack

namespace binpack {
// binpack.TightlyPack (pack_tightly.go:25-32) / binpack.DistributeEvenly (distribute_evenly.go:25-32)
inline const SparkBinPackFunction TightlyPack = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                   const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                   const resources::NodeGroupSchedulingMetadata& md) {
    return gangpack::PackOne(GP_TIGHTLY_PACK, d, e, c, dord, eord, md);
};
inline const SparkBinPackFunction DistributeEvenly = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                        const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                        const resources::NodeGroupSchedulingMetadata& md) {
    return gangpack::PackOne(GP_DISTRIBUTE_EVENLY, d, e, c, dord, eord, md);
};
// binpack.MinimalFragmentation (minimal_fragmentation.go:27-35)
inline const SparkBinPackFunction MinimalFragmentation = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                            const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                            const resources::NodeGroupSchedulingMetadata& md) {
    return gangpack::PackOne(GP_MINIMAL_FRAGMENTATION, d, e, c, dord, eord, md);
};
}  // namespace binpack

// ------------------------------------------------------------------------------------------------
// Packing efficiencies (LIB/binpack/efficiency.go) and the zone-aware tightly-pack variants
// (SURVEY §8f row f3).  Host-side float64, same operation order as the Go code; the placements
// themselves come from the device: one instance group per zone, one independent decision per zone.
namespace binpack {

struct PackingEfficiency {                 // efficiency.go:51-56
    std::string NodeName;
    double CPU = 0, Memory = 0, GPU = 0;
    double Max() const { return std::max(GPU, std::max(CPU, Memory)); }           // :59-61
};
struct AvgPackingEfficiency {              // efficiency.go:24-29
    double CPU = 0, Memory = 0, GPU = 0, Max = 0;
    bool LessThan(const AvgPackingEfficiency& o) const { return Max < o.Max; }    // :33-35
};
inline AvgPackingEfficiency WorstAvgPackingEfficiency() { return AvgPackingEfficiency{}; }   // :38-45

// Quantity.Value() of a milli-scaled CPU: whole cores, inexact values rounded away from zero
// (k8s apimachinery quantity.go:732-734 -> math.go:166-199)
inline int64_t cpuValue(int64_t milli) {
    int64_t q = milli / 1000, rem = milli % 1000;
    return rem > 0 ? q + 1 : (rem < 0 ? q - 1 : q);
}
inline int64_t normalizeResource(int64_t v) { return v == 0 ? 1 : v; }            // :104-109

// computePackingEfficiency, efficiency.go:79-102
inline PackingEfficiency computePackingEfficiency(const std::string& nodeName, const resources::NodeSchedulingMetadata& m,
                                                  const resources::NodeGroupResources& reserved) {
    resources::Resources r = m.SchedulableResources;
    r.Sub(m.AvailableResources);
    auto it = reserved.find(nodeName);
    if (it != reserved.end()) r.Add(it->second);
    PackingEfficiency e;
    e.NodeName = nodeName;
    if (m.SchedulableResources.NvidiaGPU != 0)
        e.GPU = (double)r.NvidiaGPU / (double)normalizeResource(m.SchedulableResources.NvidiaGPU);
    e.CPU = (double)cpuValue(r.CPU) / (double)normalizeResource(cpuValue(m.SchedulableResources.CPU));
    e.Memory = (double)r.Memory / (double)normalizeResource(m.SchedulableResources.Memory);
    return e;
}

// ComputeAvgPackingEfficiency, efficiency.go:114-156
inline AvgPackingEfficiency ComputeAvgPackingEfficiency(const resources::NodeGroupSchedulingMetadata& md,
                                                        const std::vector<PackingEfficiency>& effs) {
    if (effs.empty()) return WorstAvgPackingEfficiency();
    double cpuSum = 0, gpuSum = 0, memorySum = 0, maxSum = 0;
    int nodesWithGPU = 0;
    for (const auto& e : effs) {
        cpuSum += e.CPU;
        memorySum += e.Memory;
        if (md.at(e.NodeName).SchedulableResources.NvidiaGPU != 0) { gpuSum += e.GPU; nodesWithGPU++; }
        maxSum += e.Max();
    }
    double length = std::max((double)effs.size(), 1.0);
    AvgPackingEfficiency a;
    a.CPU = cpuSum / length; a.Memory = memorySum / length;
    a.GPU = nodesWithGPU == 0 ? 1.0 : gpuSum / (double)nodesWithGPU;
    a.Max = maxSum / length;
    return a;
}

// reserved map of SparkBinPack (binpack.go:72-75) rebuilt from a placement
inline resources::NodeGroupResources ReservedOf(const resources::Resources& drv, const resources::Resources& exe,
                                                const PackingResult& r) {
    resources::NodeGroupResources reserved;
    reserved[r.DriverNode] = drv;
    for (const auto& n : r.ExecutorNodes) reserved[n].Add(exe);
    return reserved;
}

// groupNodesByZone, single_az.go:57-73
inline void groupNodesByZone(const std::vector<std::string>& nodeNames, const resources::NodeGroupSchedulingMetadata& md,
                             std::vector<std::string>* zonesInOrder, std::unordered_map<std::string, std::vector<std::string>>* byZone) {
    for (const auto& n : nodeNames) {
        auto m = md.find(n);
        if (m == md.end()) continue;
        auto it = byZone->find(m->second.ZoneLabel);
        if (it == byZone->end()) { zonesInOrder->push_back(m->second.ZoneLabel); it = byZone->emplace(m->second.ZoneLabel, std::vector<std::string>{}).first; }
        it->second.push_back(n);
    }
}

using ZoneGroupList = std::vector<std::pair<std::vector<std::string>, std::vector<std::string>>>;   // (driver order, executor order)

// The candidate zones of the single-AZ packers in driverZonesInOrder order: one group per zone with both kinds of
// candidates, each holding the two orders restricted to that zone (single_az.go:30-41).
inline ZoneGroupList ZoneGroups(const std::vector<std::string>& driverOrder, const std::vector<std::string>& executorOrder,
                                const resources::NodeGroupSchedulingMetadata& md) {
    std::vector<std::string> dzOrder, ezOrder;
    std::unordered_map<std::string, std::vector<std::string>> dz, ez;
    groupNodesByZone(driverOrder, md, &dzOrder, &dz);
    groupNodesByZone(executorOrder, md, &ezOrder, &ez);
    ZoneGroupList groups;
    for (const auto& z : dzOrder)
        if (ez.count(z)) groups.emplace_back(dz[z], ez[z]);                         // :36-41
    return groups;
}

// The snapshot layout of az-aware-tightly-pack (gp_pack_batch_az_aware, gp_pack_fifo_az_aware): the candidate zones, then
// one trailing group with the nodes of both orders that no candidate zone contains -- only the undivided fallback
// (az_aware_pack_tightly.go:33-37) reaches them.  Returns the number of candidate zones.
inline int32_t AzAwareLayout(const std::vector<std::string>& driverOrder, const std::vector<std::string>& executorOrder,
                             const resources::NodeGroupSchedulingMetadata& md, ZoneGroupList* groups) {
    *groups = ZoneGroups(driverOrder, executorOrder, md);
    const int32_t nZones = (int32_t)groups->size();
    std::unordered_set<std::string> inZone;
    for (const auto& g : *groups) {
        inZone.insert(g.first.begin(), g.first.end());
        inZone.insert(g.second.begin(), g.second.end());
    }
    std::pair<std::vector<std::string>, std::vector<std::string>> rest;
    for (const auto& n : driverOrder) if (md.count(n) && !inZone.count(n)) rest.first.push_back(n);
    for (const auto& n : executorOrder) if (md.count(n) && !inZone.count(n)) rest.second.push_back(n);
    if (groups->empty() || !rest.first.empty() || !rest.second.empty()) groups->push_back(std::move(rest));
    return nZones;
}

// The undivided orders of az-aware-tightly-pack as node indices of the snapshot `d` holds (names it does not know are
// dropped, as in the groups).  eo / dord own the arrays the result points to.
inline gp_az_orders UndividedOrders(const gangpack::Device& d, int32_t nZones, const std::vector<std::string>& driverOrder,
                                    const std::vector<std::string>& executorOrder, std::vector<int32_t>* eo, std::vector<int32_t>* dord) {
    eo->clear(); dord->clear();
    for (const auto& n : executorOrder) { const int32_t i = d.index(n); if (i >= 0) eo->push_back(i); }
    for (const auto& n : driverOrder) { const int32_t i = d.index(n); if (i >= 0) dord->push_back(i); }
    gp_az_orders o{};
    o.n_zones = nZones;
    o.n_exec = (int32_t)eo->size(); o.exec_order = eo->data();
    o.n_drv = (int32_t)dord->size(); o.drv_order = dord->data();
    return o;
}

// getSingleAZSparkBinFunction(fn) + chooseBestResult, single_az.go:23-55,75-97, fn = tightlyPackExecutors or
// minimalFragmentation: every candidate zone is packed in ONE device batch (zone = instance group), the best result
// is chosen on the host by average packing efficiency over [driver] + ExecutorNodes.  The efficiencies come from
// SparkBinPack's `reserved` map (binpack.go:72-77): tightlyPackExecutors adds every executor to it,
// minimalFragmentation never touches it -> for that packer the map holds the driver only (kept as is).
inline PackingResult SingleAZPackImpl(gp_algo algo, const resources::Resources& drv, const resources::Resources& exe, int count,
                                      const std::vector<std::string>& driverOrder, const std::vector<std::string>& executorOrder,
                                      const resources::NodeGroupSchedulingMetadata& md) {
    const ZoneGroupList groups = ZoneGroups(driverOrder, executorOrder, md);
    if (groups.empty()) return EmptyPackingResult();
    gangpack::Device& d = gangpack::Device::Get();
    d.SetSnapshotGroups(md, groups);
    const size_t Z = groups.size();
    const int64_t k = count > 0 ? count : 0;
    std::vector<int64_t> dc(Z, drv.CPU), dm(Z, drv.Memory), dg(Z, drv.NvidiaGPU), ec(Z, exe.CPU), em(Z, exe.Memory), eg(Z, exe.NvidiaGPU), off(Z + 1);
    std::vector<int32_t> cnt(Z, count), grp(Z), driver(Z, -1), exec((size_t)std::max<int64_t>(k * (int64_t)Z, 1));
    for (size_t z = 0; z < Z; ++z) { grp[z] = (int32_t)z; off[z] = k * (int64_t)z; }
    off[Z] = k * (int64_t)Z;
    gp_apps a{};
    a.n_apps = (int32_t)Z;
    a.drv_cpu_milli = dc.data(); a.drv_mem_bytes = dm.data(); a.drv_gpu = dg.data();
    a.exe_cpu_milli = ec.data(); a.exe_mem_bytes = em.data(); a.exe_gpu = eg.data();
    a.exe_count = cnt.data(); a.group = grp.data(); a.exec_out_off = off.data();
    gp_results r{};
    r.driver_node = driver.data(); r.executor_nodes = exec.data(); r.executor_nodes_cap = (int64_t)exec.size();
    d.check(gp_pack_batch(d.ctx(), &a, algo, GP_MODE_INDEPENDENT, &r), "gp_pack_batch");
    PackingResult best = EmptyPackingResult();                                      // :79
    AvgPackingEfficiency bestAvg = WorstAvgPackingEfficiency();                     // :80
    for (size_t z = 0; z < Z; ++z) {
        if (driver[z] < 0) continue;                                                // :44-46
        PackingResult res;
        res.HasCapacity = true;
        res.DriverNode = d.name(driver[z]);
        for (int64_t t = off[z]; t < off[z + 1]; ++t) res.ExecutorNodes.push_back(d.name(exec[(size_t)t]));
        resources::NodeGroupResources reserved;
        if (algo == GP_MINIMAL_FRAGMENTATION) reserved[res.DriverNode] = drv;
        else reserved = ReservedOf(drv, exe, res);
        std::vector<PackingEfficiency> effs;                                        // :83-89: [driver] + executors, duplicates kept
        effs.push_back(computePackingEfficiency(res.DriverNode, md.at(res.DriverNode), reserved));
        for (const auto& n : res.ExecutorNodes) effs.push_back(computePackingEfficiency(n, md.at(n), reserved));
        AvgPackingEfficiency avg = ComputeAvgPackingEfficiency(md, effs);
        if (bestAvg.LessThan(avg)) { best = res; bestAvg = avg; }                   // :91-94
    }
    return best;
}

// AzAwareTightlyPack (az_aware_pack_tightly.go:27-38) for one application: one upload of the az-aware layout and one
// gp_pack_batch_az_aware call -- the zone packs, the zone choice and, when no zone wins, the undivided fallback all run
// on the device.
inline PackingResult AzAwarePackImpl(const resources::Resources& drv, const resources::Resources& exe, int count,
                                     const std::vector<std::string>& driverOrder, const std::vector<std::string>& executorOrder,
                                     const resources::NodeGroupSchedulingMetadata& md) {
    ZoneGroupList groups;
    const int32_t nZones = AzAwareLayout(driverOrder, executorOrder, md, &groups);
    gangpack::Device& d = gangpack::Device::Get();
    d.SetSnapshotGroups(md, groups);
    d.SetSchedulable(md);
    std::vector<int32_t> eo, dord;
    const gp_az_orders o = UndividedOrders(d, nZones, driverOrder, executorOrder, &eo, &dord);
    int64_t dc = drv.CPU, dm = drv.Memory, dg = drv.NvidiaGPU, ec = exe.CPU, em = exe.Memory, eg = exe.NvidiaGPU;
    int32_t cnt = count, zone = -1, driver = -1;
    std::vector<int32_t> exec((size_t)std::max(count, 1));
    gp_apps a{};
    a.n_apps = 1;
    a.drv_cpu_milli = &dc; a.drv_mem_bytes = &dm; a.drv_gpu = &dg;
    a.exe_cpu_milli = &ec; a.exe_mem_bytes = &em; a.exe_gpu = &eg;
    a.exe_count = &cnt;
    gp_zone_results r{};
    r.zone = &zone; r.driver_node = &driver; r.executor_nodes = exec.data(); r.executor_nodes_cap = (int64_t)exec.size();
    d.check(gp_pack_batch_az_aware(d.ctx(), &a, &o, &r), "gp_pack_batch_az_aware");
    if (driver < 0) return EmptyPackingResult();
    PackingResult res;
    res.HasCapacity = true;
    res.DriverNode = d.name(driver);
    for (int t = 0; t < count; ++t) res.ExecutorNodes.push_back(d.name(exec[(size_t)t]));
    return res;
}

inline PackingResult GuardedSingleAZ(bool azAware, const resources::Resources& d, const resources::Resources& e, int c,
                                     const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                     const resources::NodeGroupSchedulingMetadata& md, gp_algo algo = GP_TIGHTLY_PACK) {
    const int key = algo == GP_MINIMAL_FRAGMENTATION ? 102 : (azAware ? 101 : 100);
    try {
        return azAware ? AzAwarePackImpl(d, e, c, dord, eord, md) : SingleAZPackImpl(algo, d, e, c, dord, eord, md);
    } catch (const gangpack::Error&) {
        auto f = gangpack::Fallbacks().find(key);
        if (f != gangpack::Fallbacks().end() && f->second) return f->second(d, e, c, dord, eord, md);
        throw;
    }
}

// binpack.SingleAZTightlyPack (single_az_pack_tightly.go) / binpack.AzAwareTightlyPack (az_aware_pack_tightly.go:27-38)
inline const SparkBinPackFunction SingleAZTightlyPack = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                           const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                           const resources::NodeGroupSchedulingMetadata& md) {
    return GuardedSingleAZ(false, d, e, c, dord, eord, md);
};
inline const SparkBinPackFunction AzAwareTightlyPack = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                          const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                          const resources::NodeGroupSchedulingMetadata& md) {
    return GuardedSingleAZ(true, d, e, c, dord, eord, md);
};
// binpack.SingleAZMinimalFragmentation (single_az_minimal_fragmentation.go:20)
inline const SparkBinPackFunction SingleAZMinimalFragmentation = [](const resources::Resources& d, const resources::Resources& e, int c,
                                                                    const std::vector<std::string>& dord, const std::vector<std::string>& eord,
                                                                    const resources::NodeGroupSchedulingMetadata& md) {
    return GuardedSingleAZ(false, d, e, c, dord, eord, md, GP_MINIMAL_FRAGMENTATION);
};

}  // namespace binpack

// ------------------------------------------------------------------------------------------------
namespace binpacker {

struct Binpacker {                        // internal/binpacker/binpack.go:37-41
    std::string Name;
    binpack::SparkBinPackFunction BinpackFunc;
    bool IsSingleAz;
    int algo;                             // gp_algo behind BinpackFunc
};

inline const char* const tightlyPack = "tightly-pack";            // :23
inline const char* const distributeEvenly = "distribute-evenly";  // :22
inline const char* const azAwareTightlyPack = "az-aware-tightly-pack";      // :24
inline const char* const SingleAzTightlyPack = "single-az-tightly-pack";    // :29
inline const char* const SingleAzMinimalFragmentation = "single-az-minimal-fragmentation";   // :33

// binpackFunctions (:43-49): all five `binpack:` values.  `algo` is the device packer behind the function.  As a
// SparkBinPackFunction the zone-aware ones (NeedsHostLoop) choose a zone per application; extender::FitEarlierDrivers runs
// them as one device FIFO loop instead (az-aware-tightly-pack above 64 candidate zones: per driver).
inline const std::map<std::string, Binpacker>& binpackFunctions() {
    static const std::map<std::string, Binpacker> m = {
        {tightlyPack, {tightlyPack, binpack::TightlyPack, false, GP_TIGHTLY_PACK}},
        {distributeEvenly, {distributeEvenly, binpack::DistributeEvenly, false, GP_DISTRIBUTE_EVENLY}},
        {azAwareTightlyPack, {azAwareTightlyPack, binpack::AzAwareTightlyPack, false, GP_TIGHTLY_PACK}},
        {SingleAzTightlyPack, {SingleAzTightlyPack, binpack::SingleAZTightlyPack, true, GP_TIGHTLY_PACK}},
        {SingleAzMinimalFragmentation, {SingleAzMinimalFragmentation, binpack::SingleAZMinimalFragmentation, true, GP_MINIMAL_FRAGMENTATION}},
    };
    return m;
}

// packers whose placement is not ONE device packer over ONE pair of orders (they pick a zone on the host)
inline bool NeedsHostLoop(const Binpacker& b) { return b.Name != tightlyPack && b.Name != distributeEvenly; }

// SelectBinpacker (:52-58): unknown names select distribute-evenly, exactly like the reference.
inline const Binpacker* SelectBinpacker(const std::string& name) {
    auto it = binpackFunctions().find(name);
    if (it == binpackFunctions().end()) return &binpackFunctions().at(distributeEvenly);
    return &it->second;
}

}  // namespace binpacker

// ------------------------------------------------------------------------------------------------
namespace sort {

struct LabelPriorityOrder {               // config.LabelPriorityOrder, config/config.go:79-84
    std::string Name;
    std::vector<std::string> DescendingPriorityValues;
};

// NodeSorter, internal/sort/nodesorting.go:25-64.  Host-side (the step before the hot path).
class NodeSorter {
public:
    NodeSorter(const LabelPriorityOrder* driverLabel = nullptr, const LabelPriorityOrder* executorLabel = nullptr) {
        if (driverLabel) driver_ = std::make_unique<LabelPriorityOrder>(*driverLabel);
        if (executorLabel) executor_ = std::make_unique<LabelPriorityOrder>(*executorLabel);
    }

    // PotentialNodes (:41-64)
    void PotentialNodes(const resources::NodeGroupSchedulingMetadata& md, const std::vector<std::string>& nodeNames,
                        std::vector<std::string>* driverNodes, std::vector<std::string>* executorNodes) const {
        std::vector<std::string> order = getNodeNamesInPriorityOrder(md);
        std::unordered_map<std::string, int> cand;
        for (const auto& n : nodeNames) cand.emplace(n, 0);
        driverNodes->clear(); executorNodes->clear();
        for (const auto& n : order) {
            if (cand.count(n)) driverNodes->push_back(n);                                   // :52-54
            const auto& m = md.at(n);
            if (!m.Unschedulable && m.Ready) executorNodes->push_back(n);                   // :55-57
        }
        sortByLabel(*driverNodes, md, driver_.get());                                       // :61
        sortByLabel(*executorNodes, md, executor_.get());                                   // :62
    }

    // resourcesLessThan (:74-80)
    static bool resourcesLessThan(const resources::Resources& l, const resources::Resources& r) {
        if (l.Memory != r.Memory) return l.Memory < r.Memory;
        return l.CPU < r.CPU;
    }

    // getNodeNamesInPriorityOrder (:95-122); ties the reference leaves to an unstable sort are broken
    // by zone label / stable order here.
    static std::vector<std::string> getNodeNamesInPriorityOrder(const resources::NodeGroupSchedulingMetadata& md) {
        std::map<std::string, resources::Resources> az;                                     // :124-134
        for (const auto& kv : md) az[kv.second.ZoneLabel].Add(kv.second.AvailableResources);
        std::vector<std::string> labels;
        for (const auto& kv : az) labels.push_back(kv.first);
        std::stable_sort(labels.begin(), labels.end(),
                         [&](const std::string& a, const std::string& b) { return resourcesLessThan(az[a], az[b]); });  // :102-104
        std::unordered_map<std::string, int> prio;
        for (size_t i = 0; i < labels.size(); ++i) prio[labels[i]] = (int)i;
        std::vector<std::string> names;
        names.reserve(md.size());
        for (const auto& kv : md) names.push_back(kv.first);
        std::sort(names.begin(), names.end());   // deterministic starting order (Go: map order)
        std::stable_sort(names.begin(), names.end(), [&](const std::string& a, const std::string& b) {       // :83-93, :117-119
            const auto &ma = md.at(a), &mb = md.at(b);
            int pa = prio[ma.ZoneLabel], pb = prio[mb.ZoneLabel];
            if (pa != pb) return pa < pb;
            if (!ma.AvailableResources.Eq(mb.AvailableResources)) return resourcesLessThan(ma.AvailableResources, mb.AvailableResources);
            return a < b;
        });
        return names;
    }

private:
    // createLabelLessThanFunction + sortNodesByMetadataLessThanFunction (:161-200)
    static void sortByLabel(std::vector<std::string>& names, const resources::NodeGroupSchedulingMetadata& md,
                            const LabelPriorityOrder* cfg) {
        if (!cfg) return;
        std::unordered_map<std::string, int> rank;
        for (size_t i = 0; i < cfg->DescendingPriorityValues.size(); ++i) rank[cfg->DescendingPriorityValues[i]] = (int)i;
        auto rank_of = [&](const std::string& n, int* r) {
            const auto& labels = md.at(n).AllLabels;
            auto v = labels.find(cfg->Name);
            if (v == labels.end()) return false;
            auto k = rank.find(v->second);
            if (k == rank.end()) return false;
            *r = k->second;
            return true;
        };
        std::stable_sort(names.begin(), names.end(), [&](const std::string& a, const std::string& b) {
            int ra = 0, rb = 0;
            if (!rank_of(a, &ra)) return false;
            if (!rank_of(b, &rb)) return true;
            return ra < rb;
        });
    }
    std::unique_ptr<LabelPriorityOrder> driver_, executor_;
};

}  // namespace sort

// ------------------------------------------------------------------------------------------------
// ---- required node affinity (K8S = vendor/k8s.io) ---------------------------------------------------------------------
// GetRequiredNodeAffinity(pod) as strings, and their interning into gp_node_labels / gp_node_affinities: label keys and values
// become dense ids, and every rule that needs the strings is applied here -- labels.NewRequirement's validation
// (K8S/apimachinery/pkg/labels/selector.go:156-196) and the field-selector conversion (K8S/component-helpers/scheduling/corev1/
// nodeaffinity/nodeaffinity.go:203-280) become a term's parse_error flag, strconv.ParseInt of a node's label value becomes
// label_int_ok / label_int, metadata.name becomes a node index.  The same rules as affinity.encode() of the Python package.
namespace affinity {

// Requirement, Term and Program: spark_resources.hpp (a pending driver's QueuedDriverPod carries its Program)
struct Node { std::string Name; std::map<std::string, std::string> Labels; };

// strconv.ParseInt(s, 10, 64): an optional sign, then one or more ASCII digits, within int64
inline bool ParseInt(const std::string& s, int64_t* out) {
    size_t i = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0;
    if (i == s.size()) return false;
    const bool neg = s[0] == '-';
    unsigned long long v = 0;
    const unsigned long long lim = neg ? (1ull << 63) : (1ull << 63) - 1;
    for (; i < s.size(); ++i) {
        if (s[i] < '0' || s[i] > '9') return false;
        const unsigned d = (unsigned)(s[i] - '0');
        if (v > (lim - d) / 10) return false;      // out of range
        v = v * 10 + d;
    }
    *out = neg ? (int64_t)(0 - v) : (int64_t)v;
    return true;
}
inline bool AlNum(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9'); }
// ([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9], at most 63 characters
inline bool QualifiedNamePart(const std::string& s) {
    if (s.empty() || s.size() > 63 || !AlNum(s.front()) || !AlNum(s.back())) return false;
    for (char c : s) if (!AlNum(c) && c != '-' && c != '_' && c != '.') return false;
    return true;
}
// validation.IsDNS1123Subdomain: dot-separated [a-z0-9]([-a-z0-9]*[a-z0-9])?, at most 253 characters
inline bool DNS1123Subdomain(const std::string& s) {
    if (s.empty() || s.size() > 253) return false;
    size_t b = 0;
    for (;;) {
        const size_t e = std::min(s.find('.', b), s.size());
        if (e == b) return false;
        auto lower = [](char c) { return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9'); };
        if (!lower(s[b]) || !lower(s[e - 1])) return false;
        for (size_t i = b; i < e; ++i) if (!lower(s[i]) && s[i] != '-') return false;
        if (e == s.size()) return true;
        b = e + 1;
    }
}
// validation.IsQualifiedName
inline bool ValidLabelKey(const std::string& k) {
    const size_t slash = k.find('/');
    if (slash == std::string::npos) return QualifiedNamePart(k);
    if (k.find('/', slash + 1) != std::string::npos) return false;
    return DNS1123Subdomain(k.substr(0, slash)) && QualifiedNamePart(k.substr(slash + 1));
}
// validation.IsValidLabelValue
inline bool ValidLabelValue(const std::string& v) { return v.empty() || QualifiedNamePart(v); }

inline bool LabelRequirementOk(const Requirement& r) {
    static const std::set<std::string> ops = {"In", "NotIn", "Exists", "DoesNotExist", "Gt", "Lt"};
    if (!ops.count(r.Operator) || !ValidLabelKey(r.Key)) return false;
    if ((r.Operator == "In" || r.Operator == "NotIn") && r.Values.empty()) return false;
    if ((r.Operator == "Exists" || r.Operator == "DoesNotExist") && !r.Values.empty()) return false;
    int64_t v;
    if ((r.Operator == "Gt" || r.Operator == "Lt") && (r.Values.size() != 1 || !ParseInt(r.Values[0], &v))) return false;
    for (const auto& s : r.Values) if (!ValidLabelValue(s)) return false;
    return true;
}

// The arrays of gp_node_labels / gp_node_affinities; the structs point into this object
struct Encoded {
    int32_t n_nodes = 0, n_keys = 0, n_values = 0, n_aff = 0;
    std::vector<int64_t> label_off{0}, label_int, sel_off{0}, term_off{0}, term_req_off{0}, req_int, req_val_off{0};
    std::vector<int32_t> label_key, label_val, sel_key, sel_val, req_op, req_key, req_val;
    std::vector<uint8_t> label_int_ok, has_required, term_parse_error;
    gp_node_labels Labels() const {
        gp_node_labels l{};
        l.n_nodes = n_nodes; l.n_keys = n_keys; l.n_values = n_values;
        l.label_off = label_off.data(); l.label_key = label_key.data(); l.label_val = label_val.data();
        l.label_int_ok = label_int_ok.data(); l.label_int = label_int.data();
        return l;
    }
    gp_node_affinities Programs() const {
        gp_node_affinities a{};
        a.n_aff = n_aff; a.sel_off = sel_off.data(); a.sel_key = sel_key.data(); a.sel_val = sel_val.data();
        a.has_required = has_required.data(); a.term_off = term_off.data(); a.term_req_off = term_req_off.data();
        a.term_parse_error = term_parse_error.data(); a.req_op = req_op.data(); a.req_key = req_key.data(); a.req_int = req_int.data();
        a.req_val_off = req_val_off.data(); a.req_val = req_val.data();
        return a;
    }
};

template <class KeyFn, class ValFn>
inline void EncodePrograms(Encoded& e, const std::vector<Program>& programs, KeyFn key, ValFn val,
                           const std::unordered_map<std::string, int32_t>& nodeIndex);

inline Encoded Encode(const std::vector<Node>& nodes, const std::vector<Program>& programs) {
    Encoded e;
    std::unordered_map<std::string, int32_t> keys, vals, nodeIndex;
    auto key = [&](const std::string& s) { return keys.emplace(s, (int32_t)keys.size()).first->second; };
    auto val = [&](const std::string& s) { return vals.emplace(s, (int32_t)vals.size()).first->second; };
    for (size_t i = 0; i < nodes.size(); ++i)
        if (nodes[i].Name.empty() || !nodeIndex.emplace(nodes[i].Name, (int32_t)i).second)
            throw std::invalid_argument("affinity::Encode: node names must be unique and non-empty");
    for (const Node& n : nodes) {
        std::vector<std::pair<int32_t, const std::string*>> ent;
        for (const auto& kv : n.Labels) ent.emplace_back(key(kv.first), &kv.second);
        std::sort(ent.begin(), ent.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
        for (const auto& kv : ent) {
            int64_t v = 0;
            const bool ok = ParseInt(*kv.second, &v);
            e.label_key.push_back(kv.first); e.label_val.push_back(val(*kv.second));
            e.label_int_ok.push_back(ok ? 1 : 0); e.label_int.push_back(ok ? v : 0);
        }
        e.label_off.push_back((int64_t)e.label_key.size());
    }
    EncodePrograms(e, programs, key, val, nodeIndex);
    e.n_nodes = (int32_t)nodes.size(); e.n_keys = (int32_t)keys.size(); e.n_values = (int32_t)vals.size();
    return e;
}

// The gp_node_affinities arrays of the programs into e, label keys and values mapped by key / val, metadata.name by nodeIndex
template <class KeyFn, class ValFn>
inline void EncodePrograms(Encoded& e, const std::vector<Program>& programs, KeyFn key, ValFn val,
                           const std::unordered_map<std::string, int32_t>& nodeIndex) {
    auto addReq = [&](int32_t op, int32_t k, int64_t bound, std::vector<int32_t> vs) {
        std::sort(vs.begin(), vs.end());
        vs.erase(std::unique(vs.begin(), vs.end()), vs.end());
        e.req_op.push_back(op); e.req_key.push_back(k); e.req_int.push_back(bound);
        e.req_val.insert(e.req_val.end(), vs.begin(), vs.end());
        e.req_val_off.push_back((int64_t)e.req_val.size());
    };
    static const std::map<std::string, int32_t> opId = {{"In", GP_AFF_IN}, {"NotIn", GP_AFF_NOT_IN}, {"Exists", GP_AFF_EXISTS},
                                                        {"DoesNotExist", GP_AFF_DOES_NOT_EXIST}, {"Gt", GP_AFF_GT}, {"Lt", GP_AFF_LT}};
    for (const Program& p : programs) {
        for (const auto& kv : p.NodeSelector) { e.sel_key.push_back(key(kv.first)); e.sel_val.push_back(val(kv.second)); }
        e.sel_off.push_back((int64_t)e.sel_key.size());
        e.has_required.push_back(p.HasRequired ? 1 : 0);
        for (const Term& t : p.HasRequired ? p.Terms : std::vector<Term>{}) {
            bool bad = false;
            for (const auto& r : t.MatchExpressions) bad = bad || !LabelRequirementOk(r);
            for (const auto& r : t.MatchFields) bad = bad || !((r.Operator == "In" || r.Operator == "NotIn") && r.Values.size() == 1);
            e.term_parse_error.push_back(bad ? 1 : 0);
            if (!bad) {
                for (const auto& r : t.MatchExpressions) {
                    const int32_t op = opId.at(r.Operator);
                    int64_t bound = 0;
                    std::vector<int32_t> vs;
                    if (op == GP_AFF_GT || op == GP_AFF_LT) ParseInt(r.Values[0], &bound);
                    if (op == GP_AFF_IN || op == GP_AFF_NOT_IN) for (const auto& s : r.Values) vs.push_back(val(s));
                    addReq(op, key(r.Key), bound, vs);
                }
                for (const auto& r : t.MatchFields) {
                    const bool in = r.Operator == "In";
                    if (r.Key == "metadata.name") {
                        auto it = nodeIndex.find(r.Values[0]);
                        addReq(in ? GP_AFF_FIELD_NAME_IN : GP_AFF_FIELD_NAME_NOT_IN, 0, it == nodeIndex.end() ? -1 : it->second, {});
                    } else {                       // extractNodeFields sets metadata.name only: any other field reads ""
                        const bool always = (r.Values[0].empty()) == in;
                        addReq(always ? GP_AFF_FIELD_NAME_NOT_IN : GP_AFF_FIELD_NAME_IN, 0, -1, {});
                    }
                }
            }
            e.term_req_off.push_back((int64_t)e.req_op.size());
        }
        e.term_off.push_back((int64_t)e.term_parse_error.size());
    }
    e.n_aff = (int32_t)programs.size();
    // never hand a NULL pointer for an empty column
    for (auto* v : {&e.label_key, &e.label_val, &e.sel_key, &e.sel_val, &e.req_op, &e.req_key, &e.req_val}) v->reserve(1);
    for (auto* v : {&e.label_int, &e.req_int}) v->reserve(1);
    for (auto* v : {&e.label_int_ok, &e.has_required, &e.term_parse_error}) v->reserve(1);
}

// utils.ListWithPredicate(nodes, GetRequiredNodeAffinity(pod).Match) for every program at once (gp_match_node_affinity):
// matched[a] = the indices of the nodes program a matches, in node order; failed[a] = some node gave an error (the Predicate's
// failureInternal).
struct MatchResult { std::vector<std::vector<int32_t>> Matched; std::vector<bool> Failed; };
inline MatchResult MatchRequiredNodeAffinity(const std::vector<Node>& nodes, const std::vector<Program>& programs) {
    const Encoded e = Encode(nodes, programs);
    const gp_node_labels l = e.Labels();
    const gp_node_affinities a = e.Programs();
    const size_t words = (nodes.size() + 31) / 32, A = programs.size();
    std::vector<uint32_t> member(std::max<size_t>(A * words, 1));
    std::vector<int32_t> nMatch(std::max<size_t>(A, 1)), nError(std::max<size_t>(A, 1));
    gp_affinity_match out{member.data(), nMatch.data(), nError.data()};
    gangpack::Device& dev = gangpack::Device::Get();
    dev.check(gp_match_node_affinity(dev.ctx(), &l, &a, &out), "gp_match_node_affinity");
    MatchResult r;
    r.Matched.resize(A); r.Failed.resize(A);
    for (size_t p = 0; p < A; ++p) {
        r.Failed[p] = nError[p] > 0;
        for (size_t i = 0; i < nodes.size(); ++i)
            if ((member[p * words + i / 32] >> (i % 32)) & 1u) r.Matched[p].push_back((int32_t)i);
    }
    return r;
}

// Every node's labels as the resident label table (gp_label_table_*) keeps them, from the node informer: SetNode for AddFunc
// and UpdateFunc (no write when the labels are unchanged), DeleteNode for DeleteFunc.  Keys and values are interned for good,
// id 0 of each reserved for strings no node carries, so encoding a program never changes the table; node ids freed by a
// delete go to the next new node.  Flush sends what changed since the last flush in one update, after a reset with doubled
// capacities and the whole state when a capacity would be exceeded (or after Replay).
class ResidentLabels : public gangpack::ResidentTable<gp_label_table_size> {
public:
    explicit ResidentLabels(gp_label_table_size initial = {64, 16, 64, 256}) : ResidentTable(initial) {
        parsed_.push_back({0, 0});                       // value id 0: reserved
    }

    void SetNode(const Node& n) {
        auto it = labels_.find(n.Name);
        if (it != labels_.end() && it->second == n.Labels) return;
        labels_[n.Name] = n.Labels;
        auto id = nodes_.find(n.Name);
        int32_t at;
        if (id != nodes_.end()) at = id->second;
        else {
            if (!free_.empty()) { at = free_.back(); free_.pop_back(); }
            else { at = (int32_t)rows_.size(); rows_.emplace_back(); }
            nodes_.emplace(n.Name, at);
        }
        std::vector<std::pair<int32_t, int32_t>> row;
        for (const auto& kv : n.Labels) row.emplace_back(InternKey(kv.first), InternVal(kv.second));
        std::sort(row.begin(), row.end());
        rows_[(size_t)at] = std::move(row);
        dirty_.insert(at);
    }
    void DeleteNode(const std::string& name) {
        auto id = nodes_.find(name);
        if (id == nodes_.end()) return;
        rows_[(size_t)id->second].clear();
        dirty_.insert(id->second);
        free_.push_back(id->second);
        nodes_.erase(id);
        labels_.erase(name);
    }

    // the table's id of each node name, -1 for a node it does not know (no labels)
    std::vector<int32_t> NodeIDs(const std::vector<std::string>& names) const {
        std::vector<int32_t> ids(names.size(), -1);
        for (size_t i = 0; i < names.size(); ++i) {
            auto it = nodes_.find(names[i]);
            if (it != nodes_.end()) ids[i] = it->second;
        }
        return ids;
    }
    // the nodes as the per-call Encode takes them (a node the table does not know has no labels)
    std::vector<Node> Nodes(const std::vector<std::string>& names) const {
        std::vector<Node> out;
        for (const auto& nm : names) {
            auto it = labels_.find(nm);
            out.push_back(Node{nm, it == labels_.end() ? std::map<std::string, std::string>{} : it->second});
        }
        return out;
    }
    // the programs against this table's ids (gp_node_affinities of the returned object), metadata.name by index in names
    Encoded EncodePrograms(const std::vector<std::string>& names, const std::vector<Program>& programs) const {
        Encoded e;
        std::unordered_map<std::string, int32_t> nodeIndex;
        for (size_t i = 0; i < names.size(); ++i) nodeIndex.emplace(names[i], (int32_t)i);
        auto key = [&](const std::string& k) { auto it = keyId_.find(k); return it == keyId_.end() ? 0 : it->second; };
        auto val = [&](const std::string& v) { auto it = valId_.find(v); return it == valId_.end() ? 0 : it->second; };
        affinity::EncodePrograms(e, programs, key, val, nodeIndex);
        e.n_nodes = (int32_t)names.size(); e.n_keys = size_.n_keys; e.n_values = size_.n_values;
        return e;
    }

    // the id of a label key / value string; 0, the reserved id no row holds, for a string no node carries
    int32_t KeyID(const std::string& k) const { auto it = keyId_.find(k); return it == keyId_.end() ? 0 : it->second; }
    int32_t ValueID(const std::string& v) const { auto it = valId_.find(v); return it == valId_.end() ? 0 : it->second; }

    void Flush(gangpack::Device& dev) {
        int32_t longest = 0;
        for (const auto& r : rows_) longest = std::max(longest, (int32_t)r.size());
        Grow(size_.n_node_ids, (int64_t)rows_.size());
        Grow(size_.max_labels, longest);
        Grow(size_.n_keys, (int64_t)keyId_.size() + 1);
        Grow(size_.n_values, (int64_t)parsed_.size());
        std::vector<int32_t> rowNode, key, val, valueId;
        std::vector<int64_t> off{0}, valueInt;
        std::vector<uint8_t> valueOk;
        auto row = [&](int32_t at) {
            rowNode.push_back(at);
            for (const auto& kv : rows_[(size_t)at]) { key.push_back(kv.first); val.push_back(kv.second); }
            off.push_back((int64_t)key.size());
        };
        auto value = [&](int32_t v) { valueId.push_back(v); valueOk.push_back(parsed_[(size_t)v].first); valueInt.push_back(parsed_[(size_t)v].second); };
        if (Replaying()) {
            for (int32_t at = 0; at < (int32_t)rows_.size(); ++at) if (!rows_[(size_t)at].empty()) row(at);
            for (int32_t v = 1; v < (int32_t)parsed_.size(); ++v) value(v);
        } else {
            for (int32_t at : dirty_) row(at);
            for (int32_t v : newVals_) value(v);
        }
        for (auto* v : {&key, &val, &rowNode, &valueId}) v->reserve(1);
        valueOk.reserve(1); valueInt.reserve(1);
        gp_label_delta d{(int32_t)rowNode.size(), (int32_t)valueId.size(), rowNode.data(), off.data(), key.data(), val.data(),
                         valueId.data(), valueOk.data(), valueInt.data()};
        Send(dev, gp_label_table_reset, "gp_label_table_reset", gp_label_table_update, "gp_label_table_update",
             rowNode.empty() && valueId.empty() ? nullptr : &d);
        dirty_.clear();
        newVals_.clear();
    }

private:
    int32_t InternKey(const std::string& k) { return keyId_.emplace(k, (int32_t)keyId_.size() + 1).first->second; }
    int32_t InternVal(const std::string& v) {
        auto it = valId_.find(v);
        if (it != valId_.end()) return it->second;
        const int32_t id = (int32_t)parsed_.size();
        int64_t x = 0;
        const bool ok = ParseInt(v, &x);
        parsed_.push_back({ok ? 1 : 0, ok ? x : 0});
        valId_.emplace(v, id);
        newVals_.push_back(id);
        return id;
    }

    std::map<std::string, std::map<std::string, std::string>> labels_;
    std::unordered_map<std::string, int32_t> nodes_, keyId_, valId_;   // key ids start at 1, value ids at 1
    std::vector<std::pair<uint8_t, int64_t>> parsed_;             // per value id: ParseInt of the string
    std::vector<std::vector<std::pair<int32_t, int32_t>>> rows_;  // per node id: (key id, value id) by key id
    std::vector<int32_t> free_, newVals_;
    std::set<int32_t> dirty_;
};

// MatchRequiredNodeAffinity over the resident label table (gp_match_node_affinity_resident): the table's pending delta is
// flushed once, then one device call reads every label in place.  A refused call resets and replays the table and is made
// again per call, over the table's labels (Encode + gp_match_node_affinity), which answers or refuses as it does.
inline MatchResult MatchRequiredNodeAffinity(const std::vector<std::string>& nodeNames, ResidentLabels& labels,
                                             const std::vector<Program>& programs) {
    gangpack::Device& dev = gangpack::Device::Get();
    labels.Flush(dev);
    const std::vector<int32_t> ids = labels.NodeIDs(nodeNames);
    const Encoded e = labels.EncodePrograms(nodeNames, programs);
    const gp_node_affinities a = e.Programs();
    const gp_resident_labels rl{(int32_t)nodeNames.size(), 0, ids.data()};
    const size_t words = (nodeNames.size() + 31) / 32, A = programs.size();
    std::vector<uint32_t> member(std::max<size_t>(A * words, 1));
    std::vector<int32_t> nMatch(std::max<size_t>(A, 1)), nError(std::max<size_t>(A, 1));
    gp_affinity_match out{member.data(), nMatch.data(), nError.data()};
    if (gp_match_node_affinity_resident(dev.ctx(), &rl, &a, &out) != GP_OK) {
        labels.Replay();
        labels.Flush(dev);
        return MatchRequiredNodeAffinity(labels.Nodes(nodeNames), programs);
    }
    MatchResult r;
    r.Matched.resize(A); r.Failed.resize(A);
    for (size_t p = 0; p < A; ++p) {
        r.Failed[p] = nError[p] > 0;
        for (size_t i = 0; i < nodeNames.size(); ++i)
            if ((member[p * words + i / 32] >> (i % 32)) & 1u) r.Matched[p].push_back((int32_t)i);
    }
    return r;
}

}  // namespace affinity

namespace resources {

// Every node's allocatable, Spec.Unschedulable, NodeReady condition, creation time and name order as the resident node table
// (gp_node_table_*) keeps them, from the node informer: SetNode for AddFunc and UpdateFunc, after the label table's SetNode,
// which gives the node its id (no write when nothing changed); DeleteNode for DeleteFunc, before the label table's
// DeleteNode, which frees the id.  name_key is kept here: strictly increasing in the byte order of the names, in
// [0, 2^keyBits); a new name takes the midpoint of its neighbours' keys (-1 before the first, 2^keyBits after the last), and
// when no gap is left every present node gets an evenly spaced key and the next delta carries every row.  Flush sends the
// rows that differ from what the device holds as one gp_node_table_update, after a reset with a doubled capacity and the
// whole state when a node id would not fit (or after Replay, or a failed flush).
class ResidentNodes : public gangpack::ResidentTable<gp_node_table_size> {
public:
    explicit ResidentNodes(const affinity::ResidentLabels& labels, int32_t nNodeIds = 64, int keyBits = 62)
        : ResidentTable({nNodeIds, 0}), labels_(labels), keyHi_((int64_t)1 << keyBits) {}

    // creationUnixNano: metav1.Time as UnixNano (the failover reconciler's newest-first order)
    void SetNode(const std::string& name, const Resources& allocatable, bool unschedulable, bool ready, int64_t creationUnixNano = 0) {
        const int32_t at = labels_.NodeIDs({name})[0];
        if (at < 0) throw gangpack::Error(GP_ERR_INVALID, "ResidentNodes::SetNode: the label table does not know " + name + " (its SetNode first)");
        auto held = nameAt_.find(at);
        if (held != nameAt_.end() && held->second != name)
            throw gangpack::Error(GP_ERR_INVALID, "ResidentNodes::SetNode: node id held by " + held->second + " (DeleteNode it first)");
        auto cur = nodes_.find(name);
        if (cur != nodes_.end() && cur->second.id != at)
            throw gangpack::Error(GP_ERR_INVALID, "ResidentNodes::SetNode: " + name + " is held under another id (DeleteNode it before the label table's)");
        const Row row{true, {allocatable.CPU, allocatable.Memory, allocatable.NvidiaGPU}, unschedulable, ready, 0, creationUnixNano};
        if (cur != nodes_.end()) {
            Row next = row;
            next.key = cur->second.row.key;
            if (next == cur->second.row) return;
            cur->second.row = next;
        } else {
            const int64_t key = insert(name);
            Row r = row;
            r.key = key;
            nodes_[name] = Held{at, r};
            nameAt_[at] = name;
        }
        dirty_.insert(at);
    }
    void DeleteNode(const std::string& name) {
        auto it = nodes_.find(name);
        if (it == nodes_.end()) return;
        dirty_.insert(it->second.id);
        nameAt_.erase(it->second.id);
        byName_.erase(name);
        nodes_.erase(it);
    }

    // the table's id of each node name, -1 for a node it does not hold
    std::vector<int32_t> NodeIDs(const std::vector<std::string>& names) const {
        std::vector<int32_t> ids(names.size(), -1);
        for (size_t i = 0; i < names.size(); ++i) {
            auto it = nodes_.find(names[i]);
            if (it != nodes_.end()) ids[i] = it->second.id;
        }
        return ids;
    }
    int64_t NameKey(const std::string& name) const { return nodes_.at(name).row.key; }
    int Relabels() const { return relabels_; }

    // the per-call columns the node-table entries stand for: allocatable, name_rank (the byte order of the listed names, a
    // permutation of 0..n-1), unschedulable, ready and creation
    struct Columns {
        std::vector<int64_t> alloc[3];
        std::vector<int32_t> nameRank;
        std::vector<uint8_t> unschedulable, ready;
        std::vector<int64_t> creation;
    };
    Columns PerCall(const std::vector<std::string>& names) const {
        Columns c;
        std::vector<size_t> order(names.size());
        for (size_t i = 0; i < names.size(); ++i) order[i] = i;
        std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return names[a] < names[b]; });
        c.nameRank.resize(names.size());
        for (size_t r = 0; r < order.size(); ++r) c.nameRank[order[r]] = (int32_t)r;
        for (const auto& nm : names) {
            const Row& r = nodes_.at(nm).row;
            for (int d = 0; d < 3; ++d) c.alloc[d].push_back(r.alloc[d]);
            c.unschedulable.push_back(r.unschedulable);
            c.ready.push_back(r.ready);
            c.creation.push_back(r.creation);
        }
        return c;
    }

    void Flush(gangpack::Device& dev) {
        Grow(size_.n_node_ids, nameAt_.empty() ? 0 : nameAt_.rbegin()->first + 1);
        std::vector<int32_t> id;
        std::vector<uint8_t> present, uns, rdy;
        std::vector<int64_t> v[3], key, cre;
        auto row = [&](int32_t at) {
            const Row r = record(at);
            id.push_back(at); present.push_back(r.present); uns.push_back(r.unschedulable); rdy.push_back(r.ready);
            for (int d = 0; d < 3; ++d) v[d].push_back(r.alloc[d]);
            key.push_back(r.key);
            cre.push_back(r.creation);
        };
        if (Replaying()) {
            sent_.clear();
            for (const auto& kv : nameAt_) row(kv.first);
        } else {
            for (int32_t at : dirty_) {
                auto s = sent_.find(at);
                if (!(record(at) == (s == sent_.end() ? Row{} : s->second))) row(at);
            }
        }
        gp_node_delta d{(int32_t)id.size(), 0, id.data(), present.data(), v[0].data(), v[1].data(), v[2].data(), uns.data(),
                        rdy.data(), key.data(), cre.data()};
        Send(dev, gp_node_table_reset, "gp_node_table_reset", gp_node_table_update, "gp_node_table_update", id.empty() ? nullptr : &d);
        for (int32_t at : id) sent_[at] = record(at);
        dirty_.clear();
    }

private:
    struct Row {
        bool present = false;
        int64_t alloc[3] = {0, 0, 0};
        bool unschedulable = false, ready = false;
        int64_t key = 0;
        int64_t creation = 0;
        bool operator==(const Row& o) const {
            return present == o.present && alloc[0] == o.alloc[0] && alloc[1] == o.alloc[1] && alloc[2] == o.alloc[2] &&
                   unschedulable == o.unschedulable && ready == o.ready && key == o.key && creation == o.creation;
        }
    };
    struct Held { int32_t id; Row row; };

    Row record(int32_t at) const {
        auto n = nameAt_.find(at);
        return n == nameAt_.end() ? Row{} : nodes_.at(n->second).row;
    }
    // name_key of a new name (byName_ holds the present names in byte order, std::string's operator<)
    int64_t insert(const std::string& name) {
        auto next = byName_.lower_bound(name);
        const int64_t lo = next == byName_.begin() ? -1 : nodes_.at(*std::prev(next)).row.key;
        const int64_t hi = next == byName_.end() ? keyHi_ : nodes_.at(*next).row.key;
        if (hi - lo >= 2) { byName_.insert(name); return lo + (hi - lo) / 2; }
        const int64_t n = (int64_t)byName_.size() + 1, step = keyHi_ / (n + 1);
        if (step < 1) throw gangpack::Error(GP_ERR_CAPACITY, "ResidentNodes: more nodes than name keys");
        byName_.insert(name);
        int64_t j = 0, mine = 0;
        for (const auto& nm : byName_) {                // relabel: the next delta carries every row
            const int64_t k = step * ++j;
            if (nm == name) { mine = k; continue; }
            Held& h = nodes_.at(nm);
            h.row.key = k;
            dirty_.insert(h.id);
        }
        ++relabels_;
        return mine;
    }

    const affinity::ResidentLabels& labels_;
    int64_t keyHi_;
    int relabels_ = 0;
    std::unordered_map<std::string, Held> nodes_;
    std::map<int32_t, std::string> nameAt_;
    std::set<std::string> byName_;
    std::set<int32_t> dirty_;
    std::map<int32_t, Row> sent_;                 // node id -> the row the device holds
};

// The label part of a gp_node_table_nodes from the configuration's strings, against a ResidentLabels' ids: the zone label
// (failure-domain.beta.kubernetes.io/zone) with the dense zones in order and "default" appended when not listed (a node
// without the label is there, resources.go:78-81), instance-group-label with the instance groups in order, and the two
// LabelPriorityOrder's (or none).  A string no node carries gets a value id no row holds.  Decode restates the same rules on
// the label strings, for the *_resident form of the call.
struct NodeTableLabels {
    static constexpr const char* kZoneLabel = "failure-domain.beta.kubernetes.io/zone";

    NodeTableLabels(const affinity::ResidentLabels& labels, std::vector<std::string> zones, std::string instanceGroupLabel,
                    std::vector<std::string> instanceGroups, const sort::LabelPriorityOrder* driver = nullptr,
                    const sort::LabelPriorityOrder* executor = nullptr)
        : zones_(std::move(zones)), igLabel_(std::move(instanceGroupLabel)), groups_(std::move(instanceGroups)) {
        if (std::find(zones_.begin(), zones_.end(), "default") == zones_.end()) zones_.push_back("default");
        int32_t unknown = -1;
        auto ids = [&](const std::vector<std::string>& v) {
            std::vector<int32_t> out;
            for (const auto& s : v) { const int32_t x = labels.ValueID(s); out.push_back(x ? x : unknown--); }
            return out;
        };
        zoneKey_ = labels.KeyID(kZoneLabel);
        zoneValue_ = ids(zones_);
        igKey_ = labels.KeyID(igLabel_);
        igValue_ = ids(groups_);
        const sort::LabelPriorityOrder* pr[2] = {driver, executor};
        for (int k = 0; k < 2; ++k)
            if (pr[k]) { prio_[k] = *pr[k]; rankKey_[k] = labels.KeyID(pr[k]->Name); rankValue_[k] = ids(pr[k]->DescendingPriorityValues); }
    }

    void Fill(gp_node_table_nodes* n) const {
        n->zone_key = zoneKey_; n->n_zones = (int32_t)zones_.size(); n->zone_value = zoneValue_.data();
        n->zone_missing = (int32_t)(std::find(zones_.begin(), zones_.end(), "default") - zones_.begin());
        n->instance_group_key = igKey_; n->instance_group_value = igValue_.data();
        n->driver_rank_key = rankKey_[0]; n->n_driver_rank_values = (int32_t)rankValue_[0].size(); n->driver_rank_value = rankValue_[0].data();
        n->executor_rank_key = rankKey_[1]; n->n_executor_rank_values = (int32_t)rankValue_[1].size();
        n->executor_rank_value = rankValue_[1].data();
    }
    int32_t NumInstanceGroups() const { return (int32_t)groups_.size(); }
    int32_t NumZones() const { return (int32_t)zones_.size(); }

    // the per-call columns from the strings: zone (every value is listed: unknown zones are refused, false), instance group
    // (-1: none), and the label ranks (-1: extractRank's false; empty: not configured)
    struct Columns { std::vector<int32_t> zone, instanceGroup, driverRank, executorRank; };
    bool Decode(const std::vector<affinity::Node>& nodes, Columns* c) const {
        auto index = [](const std::vector<std::string>& v, const std::string& s, bool last) {
            int32_t at = -1;
            for (size_t i = 0; i < v.size(); ++i) if (v[i] == s) { at = (int32_t)i; if (!last) break; }
            return at;
        };
        for (const auto& nd : nodes) {
            auto z = nd.Labels.find(kZoneLabel);
            const int32_t zone = index(zones_, z == nd.Labels.end() ? "default" : z->second, false);
            if (zone < 0) return false;
            c->zone.push_back(zone);
            auto g = nd.Labels.find(igLabel_);
            c->instanceGroup.push_back(g == nd.Labels.end() ? -1 : index(groups_, g->second, false));
            std::vector<int32_t>* rank[2] = {&c->driverRank, &c->executorRank};
            for (int k = 0; k < 2; ++k) {
                if (rankKey_[k] < 0) continue;
                auto l = nd.Labels.find(prio_[k].Name);
                rank[k]->push_back(l == nd.Labels.end() ? -1 : index(prio_[k].DescendingPriorityValues, l->second, true));
            }
        }
        return true;
    }

private:
    std::vector<std::string> zones_;
    std::string igLabel_;
    std::vector<std::string> groups_;
    sort::LabelPriorityOrder prio_[2];
    int32_t zoneKey_ = -1, igKey_ = -1, rankKey_[2] = {-1, -1};
    std::vector<int32_t> zoneValue_, igValue_, rankValue_[2];
};

}  // namespace resources

namespace extender {

struct SparkApplicationResources {        // internal/types/types.go:22-27
    resources::Resources DriverResources;
    resources::Resources ExecutorResources;
    int MinExecutorCount = 0;
    int MaxExecutorCount = 0;
};

struct PendingDriver {                    // what fitEarlierDrivers reads off a queued driver pod
    std::string Name;
    SparkApplicationResources Resources;
    bool ParseError = false;              // sparkResources failed -> skipped (resource.go:232-237)
    bool SkipIfNoFit = false;             // shouldSkipDriverFifo (resource.go:264-270): younger than enforce-after-pod-age
};

// One queued driver pod -> what fitEarlierDrivers needs of it: sparkResources (sparkpods.go:73-137) over its annotations
// (spark_resources.hpp).  A parse error marks the entry like resource.go:232-237 does (skipped); a quantity outside the
// exact-int64 model is reported through *exact = false so that the embedding runs the original Go loop instead.
inline PendingDriver PendingDriverFromAnnotations(const std::string& name, const std::map<std::string, std::string>& annotations,
                                                  bool skipIfNoFit, bool* exact = nullptr) {
    PendingDriver d;
    d.Name = name;
    d.SkipIfNoFit = skipIfNoFit;
    ParsedSparkResources r;
    d.ParseError = !SparkResources(annotations, &r).empty();
    if (exact) *exact = r.Exact;
    if (!d.ParseError) {
        d.Resources.DriverResources = resources::CreateResources(r.DriverCPUMilli, r.DriverMemoryBytes, r.DriverNvidiaGPUs);
        d.Resources.ExecutorResources = resources::CreateResources(r.ExecutorCPUMilli, r.ExecutorMemoryBytes, r.ExecutorNvidiaGPUs);
        d.Resources.MinExecutorCount = (int)r.MinExecutorCount;
        d.Resources.MaxExecutorCount = (int)r.MaxExecutorCount;
    }
    return d;
}

// sparkResourceUsage (sparkpods.go:139-146): ASSIGNMENT semantics, kept bug-for-bug.
inline resources::NodeGroupResources SparkResourceUsage(const resources::Resources& drv, const resources::Resources& exe,
                                                        const std::string& driverNode, const std::vector<std::string>& executorNodes) {
    resources::NodeGroupResources res;
    res[driverNode] = drv;
    for (const auto& n : executorNodes) res[n] = exe;
    return res;
}

// fitEarlierDrivers (resource.go:224-262) as ONE device batch: every earlier driver is packed in queue
// order against the mutating snapshot on the GPU (GP_MODE_FIFO_REFERENCE); on return `metadata` has the
// usage of every fitted driver subtracted, exactly as the Go loop leaves it.  `results` (optional)
// receives the per-driver packing results.  Returns false when a non-skippable driver does not fit.
inline bool FitEarlierDrivers(const binpacker::Binpacker& packer, const std::vector<PendingDriver>& drivers,
                              const std::vector<std::string>& nodeNames, const std::vector<std::string>& executorNodeNames,
                              resources::NodeGroupSchedulingMetadata& metadata,
                              std::vector<binpack::PackingResult>* results = nullptr) {
    std::vector<size_t> live;   // parse errors are skipped before the packer is called (:232-237)
    for (size_t i = 0; i < drivers.size(); ++i)
        if (!drivers[i].ParseError) live.push_back(i);
    if (results) results->assign(drivers.size(), binpack::EmptyPackingResult());
    if (live.empty()) return true;
    const bool azAware = packer.Name == binpacker::azAwareTightlyPack;
    binpack::ZoneGroupList groups;
    int32_t nZones = 0;
    if (azAware) nZones = binpack::AzAwareLayout(nodeNames, executorNodeNames, metadata, &groups);
    else if (packer.IsSingleAz) {
        groups = binpack::ZoneGroups(nodeNames, executorNodeNames, metadata);
        nZones = (int32_t)groups.size();
    }
    // The single-AZ packers and az-aware-tightly-pack (up to 64 candidate zones): the whole queue in ONE launch -- zone =
    // instance group, the zone choice (or az-aware's undivided fallback) of driver i feeds driver i+1 on the device.
    // az-aware-tightly-pack with more zones keeps the per-driver loop below (gp_pack_fifo_az_aware takes at most 64).
    if (packer.IsSingleAz || (azAware && nZones <= 64)) {
        const size_t q = live.size();
        if (packer.IsSingleAz && groups.empty()) {                              // EmptyPackingResult for every driver
            for (size_t j = 0; j < q; ++j) if (!drivers[live[j]].SkipIfNoFit) return false;
            return true;
        }
        gangpack::Device& d = gangpack::Device::Get();
        d.SetSnapshotGroups(metadata, groups);
        d.SetSchedulable(metadata);
        std::vector<int64_t> dc(q), dm(q), dg(q), ec(q), em(q), eg(q);
        std::vector<int32_t> cnt(q), zone(q, -1), driver(q, -1);
        std::vector<uint8_t> skip(q);
        int64_t total = 0;
        for (size_t j = 0; j < q; ++j) {
            const auto& a = drivers[live[j]];
            dc[j] = a.Resources.DriverResources.CPU; dm[j] = a.Resources.DriverResources.Memory; dg[j] = a.Resources.DriverResources.NvidiaGPU;
            ec[j] = a.Resources.ExecutorResources.CPU; em[j] = a.Resources.ExecutorResources.Memory; eg[j] = a.Resources.ExecutorResources.NvidiaGPU;
            cnt[j] = a.Resources.MinExecutorCount;
            skip[j] = a.SkipIfNoFit ? 1 : 0;
            total += std::max(cnt[j], 0);
        }
        std::vector<int32_t> exec((size_t)std::max<int64_t>(total, 1));
        gp_apps a{};
        a.n_apps = (int32_t)q;
        a.drv_cpu_milli = dc.data(); a.drv_mem_bytes = dm.data(); a.drv_gpu = dg.data();
        a.exe_cpu_milli = ec.data(); a.exe_mem_bytes = em.data(); a.exe_gpu = eg.data();
        a.exe_count = cnt.data(); a.skip_if_no_fit = skip.data();
        gp_zone_results r{};
        r.zone = zone.data(); r.driver_node = driver.data(); r.executor_nodes = exec.data(); r.executor_nodes_cap = (int64_t)exec.size();
        if (azAware) {
            std::vector<int32_t> eo, dord;
            const gp_az_orders o = binpack::UndividedOrders(d, nZones, nodeNames, executorNodeNames, &eo, &dord);
            d.check(gp_pack_fifo_az_aware(d.ctx(), &a, GP_MODE_FIFO_REFERENCE, &o, &r), "gp_pack_fifo_az_aware");
        } else {
            d.check(gp_pack_fifo_zones(d.ctx(), &a, (gp_algo)packer.algo, GP_MODE_FIFO_REFERENCE, &r), "gp_pack_fifo_zones");
        }
        std::vector<int64_t> cpu(d.n_nodes()), mem(d.n_nodes()), gpu(d.n_nodes());
        d.check(gp_get_snapshot(d.ctx(), cpu.data(), mem.data(), gpu.data()), "gp_get_snapshot");
        for (size_t i = 0; i < d.n_nodes(); ++i) {
            auto& m = metadata.at(d.name((int32_t)i)).AvailableResources;
            m.CPU = cpu[i]; m.Memory = mem[i]; m.NvidiaGPU = gpu[i];
        }
        bool ok = true;
        int64_t at = 0;
        for (size_t j = 0; j < q; ++j) {
            if (driver[j] == -2 || (driver[j] == -1 && !skip[j])) ok = false;   // :250-252
            if (results && driver[j] >= 0) {
                auto& pr = (*results)[live[j]];
                pr.HasCapacity = true;
                pr.DriverNode = d.name(driver[j]);
                for (int64_t t = 0; t < std::max(cnt[j], 0); ++t) pr.ExecutorNodes.push_back(d.name(exec[(size_t)(at + t)]));
            }
            at += std::max(cnt[j], 0);
        }
        return ok;
    }
    if (binpacker::NeedsHostLoop(packer)) {
        // az-aware-tightly-pack with more than 64 candidate zones: the reference's own loop (:230-259), every BinpackFunc
        // call being one device batch over the zones (+ the undivided fallback); usage is subtracted on the host between
        // calls (SubtractUsageIfExists, resources.go:129-135)
        for (size_t i : live) {
            const auto& a = drivers[i];
            binpack::PackingResult pr = packer.BinpackFunc(a.Resources.DriverResources, a.Resources.ExecutorResources,
                                                           a.Resources.MinExecutorCount, nodeNames, executorNodeNames, metadata);
            if (!pr.HasCapacity) {
                if (a.SkipIfNoFit) continue;                                   // :245-249
                return false;                                                  // :250-252
            }
            for (const auto& u : SparkResourceUsage(a.Resources.DriverResources, a.Resources.ExecutorResources, pr.DriverNode, pr.ExecutorNodes)) {
                auto m = metadata.find(u.first);
                if (m != metadata.end()) m->second.AvailableResources.Sub(u.second);
            }
            if (results) (*results)[i] = pr;
        }
        return true;
    }
    gangpack::Device& d = gangpack::Device::Get();
    d.SetSnapshot(metadata, nodeNames, executorNodeNames);
    const size_t q = live.size();
    std::vector<int64_t> dc(q), dm(q), dg(q), ec(q), em(q), eg(q), off(q + 1, 0);
    std::vector<int32_t> cnt(q);
    std::vector<uint8_t> skip(q);
    for (size_t j = 0; j < q; ++j) {
        const auto& a = drivers[live[j]];
        dc[j] = a.Resources.DriverResources.CPU; dm[j] = a.Resources.DriverResources.Memory; dg[j] = a.Resources.DriverResources.NvidiaGPU;
        ec[j] = a.Resources.ExecutorResources.CPU; em[j] = a.Resources.ExecutorResources.Memory; eg[j] = a.Resources.ExecutorResources.NvidiaGPU;
        cnt[j] = a.Resources.MinExecutorCount;                     // MIN count enters the packer (:242)
        skip[j] = a.SkipIfNoFit ? 1 : 0;
        off[j + 1] = off[j] + std::max(cnt[j], 0);
    }
    std::vector<int32_t> driver(q, -1), exec((size_t)std::max<int64_t>(off[q], 1));
    gp_apps a{};
    a.n_apps = (int32_t)q;
    a.drv_cpu_milli = dc.data(); a.drv_mem_bytes = dm.data(); a.drv_gpu = dg.data();
    a.exe_cpu_milli = ec.data(); a.exe_mem_bytes = em.data(); a.exe_gpu = eg.data();
    a.exe_count = cnt.data(); a.skip_if_no_fit = skip.data(); a.exec_out_off = off.data();
    gp_results r{};
    r.driver_node = driver.data(); r.executor_nodes = exec.data(); r.executor_nodes_cap = (int64_t)exec.size();
    d.check(gp_pack_batch(d.ctx(), &a, (gp_algo)packer.algo, GP_MODE_FIFO_REFERENCE, &r), "gp_pack_batch");
    // pull the charged snapshot back into the caller's metadata (SubtractUsageIfExists, resources.go:129-135)
    std::vector<int64_t> cpu(d.n_nodes()), mem(d.n_nodes()), gpu(d.n_nodes());
    d.check(gp_get_snapshot(d.ctx(), cpu.data(), mem.data(), gpu.data()), "gp_get_snapshot");
    for (size_t i = 0; i < d.n_nodes(); ++i) {
        auto& m = metadata.at(d.name((int32_t)i)).AvailableResources;
        m.CPU = cpu[i]; m.Memory = mem[i]; m.NvidiaGPU = gpu[i];
    }
    bool ok = true;
    for (size_t j = 0; j < q; ++j) {
        if (driver[j] == -2 || (driver[j] == -1 && !skip[j])) ok = false;   // :250-252
        if (results && driver[j] >= 0) {
            auto& pr = (*results)[live[j]];
            pr.HasCapacity = true;
            pr.DriverNode = d.name(driver[j]);
            for (int64_t t = off[j]; t < off[j + 1]; ++t) pr.ExecutorNodes.push_back(d.name(exec[(size_t)t]));
        }
    }
    return ok;
}

// The node choice of rescheduleExecutor (resource.go:652-662, 675-705) on the device.  `availableNodesSchedulingMetadata`
// is the metadata of :640 (minimal-fragmentation branch), `availableResources` the map of :643 (first-fit branch),
// `overhead` the map the reference hands to GetNodeCapacities as "reserved" (:682).  Returns (node, ok) like
// rescheduleExecutorWithMinimalFragmentation; ok == false is failureFit (:672).
inline std::pair<std::string, bool> RescheduleExecutorNode(const binpacker::Binpacker& packer, const resources::Resources& executorResources,
                                                           const std::vector<std::string>& executorNodeNames,
                                                           const resources::NodeGroupSchedulingMetadata& availableNodesSchedulingMetadata,
                                                           const resources::NodeGroupResources& availableResources,
                                                           const resources::NodeGroupResources& overhead,
                                                           const std::set<std::string>& nodesWithExecutorsBelongingToThisApp) {
    gangpack::Device& d = gangpack::Device::Get();
    const bool minFrag = packer.Name == binpacker::SingleAzMinimalFragmentation;           // :652
    if (minFrag) {
        d.SetSnapshot(availableNodesSchedulingMetadata, {}, executorNodeNames);
    } else {
        resources::NodeGroupSchedulingMetadata md;
        for (const auto& kv : availableResources) md[kv.first].AvailableResources = kv.second;
        d.SetSnapshot(md, {}, executorNodeNames);
    }
    const size_t N = d.n_nodes();
    int64_t ec = executorResources.CPU, em = executorResources.Memory, eg = executorResources.NvidiaGPU;
    std::vector<int64_t> rc(N, 0), rm(N, 0), rg(N, 0);
    std::vector<int32_t> hosting;
    int64_t hoff[2] = {0, 0};
    gp_reschedule in{};
    in.n_execs = 1; in.exe_cpu_milli = &ec; in.exe_mem_bytes = &em; in.exe_gpu = &eg; in.min_frag = minFrag ? 1 : 0;
    if (minFrag) {
        for (const auto& kv : overhead) {
            int32_t i = d.index(kv.first);
            if (i >= 0) { rc[(size_t)i] = kv.second.CPU; rm[(size_t)i] = kv.second.Memory; rg[(size_t)i] = kv.second.NvidiaGPU; }
        }
        for (const auto& n : nodesWithExecutorsBelongingToThisApp) { int32_t i = d.index(n); if (i >= 0) hosting.push_back(i); }
        hoff[1] = (int64_t)hosting.size();
        in.reserved_cpu_milli = rc.data(); in.reserved_mem_bytes = rm.data(); in.reserved_gpu = rg.data();
        in.host_off = hoff; in.host_nodes = hosting.data();
    }
    int32_t node = -1;
    if (N == 0) return {std::string(), false};
    d.check(gp_reschedule_executors(d.ctx(), &in, &node), "gp_reschedule_executors");
    if (node < 0) return {std::string(), false};
    return {d.name(node), true};
}

// computeAvgPackingEfficiencyForResult (internal/extender/resource.go:372-381): the Predicate's packing-efficiency metric,
// ComputeAvgPackingEfficiency over the PackingEfficiencies of EVERY node of nodesSchedulingMetadata, with `reserved` rebuilt
// from the placement (binpack.go:72-77: driver + every executor; minimal-fragmentation -- algo GP_MINIMAL_FRAGMENTATION,
// also for single-az-minimal-fragmentation winners -- the driver only).  Computed by one gp_packing_efficiency call; its
// sums are rounded once from their exact value, so it agrees with the Go loop (map order) within the recursive-summation
// bound and bit for bit where every partial sum is exact.  The Go function reads packingResult.PackingEfficiencies; this
// layer's PackingResult does not carry them, so the resources of the placed application are passed instead.
// EmptyPackingResult -> WorstAvgPackingEfficiency.
inline binpack::AvgPackingEfficiency ComputeAvgPackingEfficiencyForResult(const resources::NodeGroupSchedulingMetadata& nodesSchedulingMetadata,
                                                                           const binpack::PackingResult& packingResult,
                                                                           const resources::Resources& driverResources,
                                                                           const resources::Resources& executorResources,
                                                                           gp_algo algo = GP_TIGHTLY_PACK) {
    if (!packingResult.HasCapacity) return binpack::WorstAvgPackingEfficiency();
    gangpack::Device& d = gangpack::Device::Get();
    d.SetSnapshotAll(nodesSchedulingMetadata);
    auto idx = [&](const std::string& n) {
        const int32_t i = d.index(n);
        if (i < 0) throw gangpack::Error(GP_ERR_INVALID, "ComputeAvgPackingEfficiencyForResult: node not in the metadata: " + n);
        return i;
    };
    int32_t driver = idx(packingResult.DriverNode);
    std::vector<int32_t> execs;
    for (const auto& n : packingResult.ExecutorNodes) execs.push_back(idx(n));
    const int32_t count = (int32_t)execs.size();
    if (execs.empty()) execs.push_back(0);
    const int64_t drv[3] = {driverResources.CPU, driverResources.Memory, driverResources.NvidiaGPU};
    const int64_t exe[3] = {executorResources.CPU, executorResources.Memory, executorResources.NvidiaGPU};
    const int64_t off[2] = {0, count};
    gp_apps a{};
    a.n_apps = 1;
    a.drv_cpu_milli = &drv[0]; a.drv_mem_bytes = &drv[1]; a.drv_gpu = &drv[2];
    a.exe_cpu_milli = &exe[0]; a.exe_mem_bytes = &exe[1]; a.exe_gpu = &exe[2];
    a.exe_count = &count; a.exec_out_off = off;
    gp_results r{&driver, execs.data(), (int64_t)execs.size()};
    double avg[4] = {0, 0, 0, 0};
    d.check(gp_packing_efficiency(d.ctx(), &a, algo, &r, GP_MODE_INDEPENDENT, avg), "gp_packing_efficiency");
    binpack::AvgPackingEfficiency out;
    out.CPU = avg[0]; out.Memory = avg[1]; out.GPU = avg[2]; out.Max = avg[3];
    return out;
}

// The two zone labels rescheduleExecutor reads, and they differ (SURVEY App. B5): PotentialNodes sorts by
// NodeSchedulingMetadata.ZoneLabel, the BETA label with the placeholder "default" when it is absent
// (LIB/resources/resources.go:27,78-81); filterNodesToZone and getAzsOfPods read the GA label (resource.go:466,526).
inline const char* const LabelZoneFailureDomain = "failure-domain.beta.kubernetes.io/zone";   // corev1.LabelZoneFailureDomain
inline const char* const LabelTopologyZone = "topology.kubernetes.io/zone";                   // v1.LabelTopologyZone

// One node of availableNodes (getNodes(nodeNames), resource.go:604) as rescheduleExecutor reads it.
struct RescheduleNode {
    std::string Name;
    resources::Resources Allocatable;                  // node.Status.Allocatable
    bool Unschedulable = false;
    bool Ready = true;
    std::map<std::string, std::string> AllLabels;      // node.Labels: both zone labels and the executor label priority
};
struct ReservationRow {                                // one hard or soft reservation (GetReservedResources, resourcereservations.go:258-263)
    std::string Node;
    resources::Resources Resources;
};
struct RescheduleOutcome {
    std::string Node;                                  // chosen node, "" = failureFit (:672)
    bool Found = false;
    bool Ambiguous = false;                            // the reference's own choice is unspecified (SURVEY App. B6)
};

// rescheduleExecutor (resource.go:594-673) minus pod and lister I/O, in ONE device call (gp_reschedule_from_reservations):
// GetReservedResources -> NodeSchedulingMetadataForNodes -> AvailableForNodes (overhead counted twice, App. B7) ->
// PotentialNodes -> first fit or rescheduleExecutorWithMinimalFragmentation.  commonZone: the zone
// getCommonZoneForExecutorsApplication returned (filterNodesToZone then runs first over LabelTopologyZone; a node without that
// label throws, as the reference errors), or nullptr.  The executor order's zone priority comes from LabelZoneFailureDomain
// ("default" when absent), as in the reference.  The device context's resident snapshot is not touched.
inline RescheduleOutcome RescheduleExecutor(const binpacker::Binpacker& packer, const resources::Resources& executorResources,
                                            const std::vector<RescheduleNode>& availableNodes, const std::vector<ReservationRow>& reservations,
                                            const resources::NodeGroupResources& overhead, const sort::LabelPriorityOrder* executorLabel,
                                            const std::string* commonZone,
                                            const std::set<std::string>& nodesWithExecutorsBelongingToThisApp) {
    RescheduleOutcome out;
    const size_t N = availableNodes.size();
    if (N == 0) return out;
    std::unordered_map<std::string, int32_t> index, zoneId, topoId;   // sorter zones and topology zones, interned separately
    std::vector<int64_t> ac(N), am(N), ag(N), oc(N, 0), om(N, 0), og(N, 0);
    std::vector<int32_t> zone(N), topo(N), nameRank(N), labelRank(N, -1);
    std::vector<uint8_t> unsched(N), ready(N);
    std::unordered_map<std::string, int> rankOfValue;
    if (executorLabel)
        for (size_t i = 0; i < executorLabel->DescendingPriorityValues.size(); ++i) rankOfValue[executorLabel->DescendingPriorityValues[i]] = (int)i;
    for (size_t i = 0; i < N; ++i) {
        const RescheduleNode& n = availableNodes[i];
        index[n.Name] = (int32_t)i;
        ac[i] = n.Allocatable.CPU; am[i] = n.Allocatable.Memory; ag[i] = n.Allocatable.NvidiaGPU;
        auto o = overhead.find(n.Name);                                                   // GetOverhead(availableNodes)
        if (o != overhead.end()) { oc[i] = o->second.CPU; om[i] = o->second.Memory; og[i] = o->second.NvidiaGPU; }
        auto beta = n.AllLabels.find(LabelZoneFailureDomain);                            // the sorter's zone (resources.go:78-81)
        const std::string& sortZone = beta == n.AllLabels.end() ? std::string("default") : beta->second;
        zone[i] = zoneId.emplace(sortZone, (int32_t)zoneId.size()).first->second;       // interned in first-seen order
        auto ga = n.AllLabels.find(LabelTopologyZone);                                  // filterNodesToZone's label (:466)
        topo[i] = ga == n.AllLabels.end() ? -1 : topoId.emplace(ga->second, (int32_t)topoId.size()).first->second;
        unsched[i] = n.Unschedulable ? 1 : 0; ready[i] = n.Ready ? 1 : 0;
        if (executorLabel) {
            auto v = n.AllLabels.find(executorLabel->Name);
            if (v != n.AllLabels.end()) { auto r = rankOfValue.find(v->second); if (r != rankOfValue.end()) labelRank[i] = r->second; }
        }
    }
    std::vector<size_t> byName(N);
    for (size_t i = 0; i < N; ++i) byName[i] = i;
    std::sort(byName.begin(), byName.end(), [&](size_t a, size_t b) { return availableNodes[a].Name < availableNodes[b].Name; });
    for (size_t r = 0; r < N; ++r) nameRank[byName[r]] = (int32_t)r;
    std::vector<int32_t> rn;
    std::vector<int64_t> rc, rm, rg;
    rn.reserve(reservations.size()); rc.reserve(reservations.size()); rm.reserve(reservations.size()); rg.reserve(reservations.size());
    for (const auto& r : reservations) {
        auto it = index.find(r.Node);
        rn.push_back(it == index.end() ? -1 : it->second);                                // not in the table: ignored (resources.go:72-75)
        rc.push_back(r.Resources.CPU); rm.push_back(r.Resources.Memory); rg.push_back(r.Resources.NvidiaGPU);
    }
    gp_usage_input u{};
    u.n_nodes = (int32_t)N;
    u.alloc_cpu_milli = ac.data(); u.alloc_mem_bytes = am.data(); u.alloc_gpu = ag.data();
    u.overhead_cpu_milli = oc.data(); u.overhead_mem_bytes = om.data(); u.overhead_gpu = og.data();
    u.n_reservations = (int64_t)rn.size();
    u.res_node = rn.data(); u.res_cpu_milli = rc.data(); u.res_mem_bytes = rm.data(); u.res_gpu = rg.data();
    gp_sort_input s{};
    s.n_nodes = (int32_t)N;
    s.n_zones = (int32_t)zoneId.size();
    s.zone_id = zone.data(); s.name_rank = nameRank.data(); s.unschedulable = unsched.data(); s.ready = ready.data();
    s.executor_label_rank = executorLabel ? labelRank.data() : nullptr;
    gp_reschedule_scope scope{};
    scope.keep_topology_zone = -1;
    scope.topology_zone = topo.data();
    if (commonZone) {
        auto z = topoId.find(*commonZone);
        scope.keep_topology_zone = z == topoId.end() ? (int32_t)topoId.size() : z->second;   // a zone no node has: nothing kept
    }
    const bool minFrag = packer.Name == binpacker::SingleAzMinimalFragmentation;             // :652
    int64_t ec = executorResources.CPU, em = executorResources.Memory, eg = executorResources.NvidiaGPU;
    std::vector<int32_t> hosting;
    for (const auto& n : nodesWithExecutorsBelongingToThisApp) { auto it = index.find(n); if (it != index.end()) hosting.push_back(it->second); }
    int64_t hoff[2] = {0, (int64_t)hosting.size()};
    gp_reschedule in{};
    in.n_execs = 1; in.exe_cpu_milli = &ec; in.exe_mem_bytes = &em; in.exe_gpu = &eg; in.min_frag = minFrag ? 1 : 0;
    if (minFrag) { in.host_off = hoff; in.host_nodes = hosting.data(); }
    int32_t node = -1;
    uint8_t ambiguous = 0;
    gangpack::Device& d = gangpack::Device::Get();
    d.check(gp_reschedule_from_reservations(d.ctx(), &u, &s, commonZone ? &scope : nullptr, &in, &node, &ambiguous),
            "gp_reschedule_from_reservations");
    out.Ambiguous = ambiguous != 0;
    if (node >= 0) { out.Node = availableNodes[(size_t)node].Name; out.Found = true; }
    return out;
}

class ResidentOverheadComputer;
class ResidentDrivers;

// The unschedulable-pod marker's capacity checks (scanForUnschedulablePods, internal/extender/unschedulablepods.go:93-129) for
// ALL stale drivers in one device call (gp_exceeds_cluster_capacity) instead of one DoesPodExceedClusterCapacity (:132-166) each.
class UnschedulablePodMarker {
public:
    struct CapacityNode {              // what the resident sweep reads of a node: allocatable and zone, the overhead is the table's
        std::string Name;
        resources::Resources Allocatable;
        std::string ZoneLabel = "default";
    };
    struct StaleDriver {
        resources::Resources DriverResources;
        resources::Resources ExecutorResources;
        int MinExecutorCount = 0;
        int AffinityClass = -1;        // index into the caller's affinity classes; -1 = the required affinity matches every node
    };
    explicit UnschedulablePodMarker(const binpacker::Binpacker& packer) : packer_(packer) {}

    // nodesSchedulingMetadata: NodeSchedulingMetadataForNodes(every node, zero usage, GetNonSchedulableOverhead) -- only
    // SchedulableResources and ZoneLabel are read.  nodeClass: the affinity class of each node (absent = in none);
    // nClasses: the number of classes.  -> exceeds[i] for drivers[i].  The device context's resident snapshot is not touched.
    std::vector<bool> DoesPodsExceedClusterCapacity(const resources::NodeGroupSchedulingMetadata& nodesSchedulingMetadata,
                                                    const std::unordered_map<std::string, int32_t>& nodeClass, int32_t nClasses,
                                                    const std::vector<StaleDriver>& drivers) const {
        const size_t N = nodesSchedulingMetadata.size(), Q = drivers.size();
        std::vector<int64_t> sc, sm, sg;
        std::vector<int32_t> zone, group;
        sc.reserve(N); sm.reserve(N); sg.reserve(N); zone.reserve(N); group.reserve(N);
        std::unordered_map<std::string, int32_t> zoneId;
        for (const auto& kv : nodesSchedulingMetadata) {
            const auto& s = kv.second.SchedulableResources;
            sc.push_back(s.CPU); sm.push_back(s.Memory); sg.push_back(s.NvidiaGPU);
            zone.push_back(zoneId.emplace(kv.second.ZoneLabel, (int32_t)zoneId.size()).first->second);
            auto c = nodeClass.find(kv.first);
            group.push_back(c == nodeClass.end() ? -1 : c->second);
        }
        std::vector<int64_t> q[6];
        std::vector<int32_t> count(Q), cls(Q);
        for (auto& col : q) col.resize(Q);
        for (size_t i = 0; i < Q; ++i) {
            const StaleDriver& d = drivers[i];
            q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
            q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
            count[i] = d.MinExecutorCount; cls[i] = d.AffinityClass;
        }
        gp_capacity_nodes n{};
        n.n_nodes = (int32_t)N;
        n.alloc_cpu_milli = sc.data(); n.alloc_mem_bytes = sm.data(); n.alloc_gpu = sg.data();   // schedulable = alloc - overhead
        n.n_zones = std::max<int32_t>(1, (int32_t)zoneId.size()); n.zone_id = zone.data();
        n.n_groups = std::max<int32_t>(1, nClasses); n.node_group = group.data();
        gp_apps a{};
        a.n_apps = (int32_t)Q;
        a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
        a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
        a.exe_count = count.data(); a.group = cls.data();
        std::vector<uint8_t> out(std::max<size_t>(Q, 1));
        gangpack::Device& dev = gangpack::Device::Get();
        dev.check(gp_exceeds_cluster_capacity(dev.ctx(), &n, &a, Packer(), out.data()), "gp_exceeds_cluster_capacity");
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    }

    // The same sweep with GetNonSchedulableOverhead read in place from the resident overhead table: the table's pending delta
    // is flushed once, then one gp_exceeds_cluster_capacity_resident call.  A refused call resets and replays the table and
    // is made again per call, over GetNonSchedulableOverhead (defined after ResidentOverheadComputer).
    std::vector<bool> DoesPodsExceedClusterCapacity(const std::vector<CapacityNode>& nodes, ResidentOverheadComputer& overhead,
                                                    const std::unordered_map<std::string, int32_t>& nodeClass, int32_t nClasses,
                                                    const std::vector<StaleDriver>& drivers) const;

    // The same sweep with each driver's node set = the nodes its required affinity matches (gp_exceeds_cluster_capacity_affinity):
    // the sets may overlap freely.  nodes: the node table with labels, every node in nodesSchedulingMetadata; programs: one
    // per distinct required affinity; drivers[i].Affinity indexes programs.  affinityError[i] = ListWithPredicate failed for
    // driver i's affinity (the reference's scan returns at that driver, unschedulablepods.go:113-117); exceeds[i] is then
    // meaningless.
    struct AffinityStaleDriver {
        resources::Resources DriverResources;
        resources::Resources ExecutorResources;
        int MinExecutorCount = 0;
        int Affinity = 0;              // index into programs
    };
    std::vector<bool> DoesPodsExceedClusterCapacity(const resources::NodeGroupSchedulingMetadata& nodesSchedulingMetadata,
                                                    const std::vector<affinity::Node>& nodes,
                                                    const std::vector<affinity::Program>& programs,
                                                    const std::vector<AffinityStaleDriver>& drivers,
                                                    std::vector<bool>* affinityError) const {
        const size_t N = nodes.size(), Q = drivers.size();
        std::vector<int64_t> sc(N + 1), sm(N + 1), sg(N + 1);
        std::vector<int32_t> zone(N + 1);
        std::unordered_map<std::string, int32_t> zoneId;
        for (size_t i = 0; i < N; ++i) {
            const auto& m = nodesSchedulingMetadata.at(nodes[i].Name);
            sc[i] = m.SchedulableResources.CPU; sm[i] = m.SchedulableResources.Memory; sg[i] = m.SchedulableResources.NvidiaGPU;
            zone[i] = zoneId.emplace(m.ZoneLabel, (int32_t)zoneId.size()).first->second;
        }
        std::vector<int64_t> q[6];
        std::vector<int32_t> count(Q + 1), prog(Q + 1);
        for (auto& col : q) col.resize(Q + 1);
        for (size_t i = 0; i < Q; ++i) {
            const AffinityStaleDriver& d = drivers[i];
            q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
            q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
            count[i] = d.MinExecutorCount; prog[i] = d.Affinity;
        }
        const affinity::Encoded e = affinity::Encode(nodes, programs);
        const gp_node_labels l = e.Labels();
        const gp_node_affinities p = e.Programs();
        gp_capacity_nodes n{};
        n.n_nodes = (int32_t)N;
        n.alloc_cpu_milli = sc.data(); n.alloc_mem_bytes = sm.data(); n.alloc_gpu = sg.data();   // schedulable = alloc - overhead
        n.n_zones = std::max<int32_t>(1, (int32_t)zoneId.size()); n.zone_id = zone.data();
        gp_apps a{};
        a.n_apps = (int32_t)Q;
        a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
        a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
        a.exe_count = count.data(); a.group = prog.data();
        std::vector<uint8_t> out(Q + 1), err(Q + 1);
        gangpack::Device& dev = gangpack::Device::Get();
        dev.check(gp_exceeds_cluster_capacity_affinity(dev.ctx(), &n, &l, &p, &a, Packer(), out.data(), err.data()),
                  "gp_exceeds_cluster_capacity_affinity");
        if (affinityError) affinityError->assign(err.begin(), err.begin() + (std::ptrdiff_t)Q);
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    }

    // The affinity sweep over both resident tables: GetNonSchedulableOverhead from the overhead table and every node's labels
    // from the label table, each flushed once, then one gp_exceeds_cluster_capacity_affinity_label_table call.  A refused
    // call resets and replays both tables and is made again per call, over the tables' labels and GetNonSchedulableOverhead
    // (defined after ResidentOverheadComputer).
    std::vector<bool> DoesPodsExceedClusterCapacity(const std::vector<CapacityNode>& nodes, ResidentOverheadComputer& overhead,
                                                    affinity::ResidentLabels& labels, const std::vector<affinity::Program>& programs,
                                                    const std::vector<AffinityStaleDriver>& drivers, std::vector<bool>* affinityError) const;

    // The two resident sweeps with allocatable from the node table and the zone from the label table: names lists the nodes,
    // zones the dense zones ("default" appended when not listed).  The overhead, label and node tables are flushed once,
    // then one gp_exceeds_cluster_capacity[_affinity]_node_table call.  A refused call resets and replays the three tables and
    // makes the resident sweep above over the columns the host decodes from them (defined after ResidentOverheadComputer).
    std::vector<bool> DoesPodsExceedClusterCapacity(const std::vector<std::string>& names, resources::ResidentNodes& nodes,
                                                    affinity::ResidentLabels& labels, ResidentOverheadComputer& overhead,
                                                    const std::vector<std::string>& zones,
                                                    const std::unordered_map<std::string, int32_t>& nodeClass, int32_t nClasses,
                                                    const std::vector<StaleDriver>& drivers) const;
    std::vector<bool> DoesPodsExceedClusterCapacity(const std::vector<std::string>& names, resources::ResidentNodes& nodes,
                                                    affinity::ResidentLabels& labels, ResidentOverheadComputer& overhead,
                                                    const std::vector<std::string>& zones, const std::vector<affinity::Program>& programs,
                                                    const std::vector<AffinityStaleDriver>& drivers, std::vector<bool>* affinityError) const;

    // The whole scan from the resident driver table too (gp_exceeds_cluster_capacity_driver_table): the stale drivers of
    // schedulerName (creation + timeout < now) are selected, ordered by (creation, slot) and checked on the device against
    // each one's required affinity, which the driver table interns.  The overhead, label, node and driver tables are flushed
    // once, then one call; a capacity refusal grows the output and calls again.  Any other refusal replays the four tables
    // and answers with the per-call node-table affinity sweep above over the stale drivers decoded from the held pods.
    // -> one entry per stale driver: Outcome 0 answered (Exceeds), 1 its affinity errors (ListWithPredicate fails), 2 outside
    // the exact-int64 model (inexact, a negative quantity or count: the caller answers it with DoesPodExceedClusterCapacity).
    struct StaleOutcome {
        std::string UID;
        bool Exceeds = false;
        int32_t Outcome = 0;
    };
    std::vector<StaleOutcome> DoesPodsExceedClusterCapacity(ResidentDrivers& drivers, const std::string& schedulerName, int64_t timeoutNs,
                                                            int64_t nowUnixNano, const std::vector<std::string>& names,
                                                            resources::ResidentNodes& nodes, affinity::ResidentLabels& labels,
                                                            ResidentOverheadComputer& overhead, const std::vector<std::string>& zones) const;
    // true when the last driver-table scan was answered by the per-call path
    bool LastScanFellBack() const { return fellBack_; }

private:
    gp_binpacker Packer() const {
        if (packer_.Name == binpacker::tightlyPack) return GP_BP_TIGHTLY_PACK;
        if (packer_.Name == binpacker::azAwareTightlyPack) return GP_BP_AZ_AWARE_TIGHTLY_PACK;
        if (packer_.Name == binpacker::SingleAzTightlyPack) return GP_BP_SINGLE_AZ_TIGHTLY_PACK;
        if (packer_.Name == binpacker::SingleAzMinimalFragmentation) return GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION;
        return GP_BP_DISTRIBUTE_EVENLY;                 // SelectBinpacker's default
    }
    binpacker::Binpacker packer_;
    mutable int32_t staleCap_ = 64;                    // the driver-table scan's output size, grown on a capacity refusal
    mutable bool fellBack_ = false;
};

// The failover reconciler's node choice (syncResourceReservationsAndDemands, internal/extender/failover.go:43-82):
// availableResourcesPerInstanceGroup (:286-323) and, per stale driver, constructResourceReservation's findNodes (:348-390,
// 409-436) with the charge of :159 -- one gp_reconcile_find_nodes call for every stale driver.  Pod and reservation listing,
// the RR writes and syncDemands / syncSoftReservations stay with the caller.
struct ReconcileNode {
    std::string Name;
    resources::Resources Allocatable;
    std::unordered_map<std::string, std::string> Labels;
    bool Unschedulable = false;
    bool Ready = true;
    int64_t CreationUnixNano = 0;          // metav1.Time, ordered like Before
};
struct ReconcileRow {                      // one RR reservation or one soft reservation
    std::string Node;
    resources::Resources Resources;
};
struct StaleDriver {
    std::string InstanceGroup;             // FindInstanceGroupFromPodSpec; "" when the driver names none
    resources::Resources ExecutorResources;
    int MinExecutorCount = 0;
    int RunningExecutors = 0;              // inconsistent executors already running; capped at MinExecutorCount (:141-143)
};
struct ReconcileResult {
    bool InstanceGroupFound = false;       // false: constructResourceReservation errs (:358-362) and nothing is charged
    std::vector<std::string> ReservedNodeNames;
};

// The node table (minus its usage) and the stale drivers of one reconcile as gp_reconcile_find_nodes[_resident] take them,
// and the results read back.  Holds pointers into its own vectors: not copied.
struct ReconcileCall {
    std::vector<int64_t> ac, am, ag, cr, ec, em, eg, off;
    std::vector<int32_t> grp, count, dg, placed, exe;
    std::vector<uint8_t> unsched, ready;
    gp_reconcile_nodes nd{};
    gp_apps a{};
    gp_reconcile_results out{};
    // groups (or NULL): instance-group values that take ids 0, 1, .. before any node's or driver's
    ReconcileCall(const std::vector<ReconcileNode>& nodes, const std::string& instanceGroupLabel, const std::vector<StaleDriver>& drivers,
                  const std::vector<std::string>* groups = nullptr) {
        const size_t N = nodes.size(), Q = drivers.size();
        std::unordered_map<std::string, int32_t> groupId;
        auto intern = [&](const std::string& g) { return groupId.emplace(g, (int32_t)groupId.size()).first->second; };
        if (groups) for (const auto& g : *groups) intern(g);
        ac.resize(N); am.resize(N); ag.resize(N); cr.resize(N); grp.resize(N); unsched.resize(N); ready.resize(N);
        for (size_t i = 0; i < N; ++i) {
            const ReconcileNode& n = nodes[i];
            ac[i] = n.Allocatable.CPU; am[i] = n.Allocatable.Memory; ag[i] = n.Allocatable.NvidiaGPU;
            auto l = n.Labels.find(instanceGroupLabel);
            grp[i] = intern(l == n.Labels.end() ? std::string() : l->second);      // n.Labels[label]: "" when missing
            unsched[i] = n.Unschedulable; ready[i] = n.Ready; cr[i] = n.CreationUnixNano;
        }
        ec.resize(Q); em.resize(Q); eg.resize(Q); off.assign(Q + 1, 0); count.resize(Q); dg.resize(Q);
        for (size_t i = 0; i < Q; ++i) {
            const StaleDriver& d = drivers[i];
            ec[i] = d.ExecutorResources.CPU; em[i] = d.ExecutorResources.Memory; eg[i] = d.ExecutorResources.NvidiaGPU;
            count[i] = std::max(0, d.MinExecutorCount - std::min(d.RunningExecutors, d.MinExecutorCount));   // :366
            dg[i] = intern(d.InstanceGroup);
            off[i + 1] = off[i] + count[i];
        }
        nd.n_groups = std::max<int32_t>(1, (int32_t)groupId.size());
        nd.node_group = grp.data(); nd.creation = cr.data(); nd.unschedulable = unsched.data(); nd.ready = ready.data();
        a.n_apps = (int32_t)Q;
        a.exe_cpu_milli = ec.data(); a.exe_mem_bytes = em.data(); a.exe_gpu = eg.data();
        a.exe_count = count.data(); a.group = dg.data(); a.exec_out_off = off.data();
        placed.resize(std::max<size_t>(Q, 1)); exe.resize((size_t)std::max<int64_t>(off[Q], 1));
        out.placed = placed.data(); out.executor_nodes = exe.data(); out.executor_nodes_cap = off[Q];
    }
    ReconcileCall(const ReconcileCall&) = delete;
    ReconcileCall& operator=(const ReconcileCall&) = delete;
    std::vector<ReconcileResult> Results(const std::vector<ReconcileNode>& nodes) const {
        std::vector<std::string> names;
        for (const auto& n : nodes) names.push_back(n.Name);
        return Results(names);
    }
    std::vector<ReconcileResult> Results(const std::vector<std::string>& names) const {
        std::vector<ReconcileResult> res((size_t)a.n_apps);
        for (size_t i = 0; i < res.size(); ++i) {
            res[i].InstanceGroupFound = placed[i] >= 0;
            for (int32_t j = 0; j < placed[i]; ++j) res[i].ReservedNodeNames.push_back(names[(size_t)exe[(size_t)off[i] + (size_t)j]]);
        }
        return res;
    }
};

// nodes: the lister's nodes (their order is the tie order among equal creation times, DESIGN §2.3); rows: every RR and soft
// reservation; overhead: GetOverhead by node name; drivers: in the order their RRs are written.
inline std::vector<ReconcileResult> ReconcileFindNodes(const std::vector<ReconcileNode>& nodes, const std::vector<ReconcileRow>& rows,
                                                       const resources::NodeGroupResources& overhead, const std::string& instanceGroupLabel,
                                                       const std::vector<StaleDriver>& drivers) {
    const size_t N = nodes.size(), R = rows.size();
    ReconcileCall call(nodes, instanceGroupLabel, drivers);
    std::unordered_map<std::string, int32_t> index;
    std::vector<int64_t> oc(N), om(N), og(N);
    for (size_t i = 0; i < N; ++i) {
        index.emplace(nodes[i].Name, (int32_t)i);
        auto o = overhead.find(nodes[i].Name);
        if (o != overhead.end()) { oc[i] = o->second.CPU; om[i] = o->second.Memory; og[i] = o->second.NvidiaGPU; }
    }
    std::vector<int32_t> rn(R);
    std::vector<int64_t> rc(R), rm(R), rg(R);
    for (size_t r = 0; r < R; ++r) {
        auto it = index.find(rows[r].Node);
        rn[r] = it == index.end() ? -1 : it->second;
        rc[r] = rows[r].Resources.CPU; rm[r] = rows[r].Resources.Memory; rg[r] = rows[r].Resources.NvidiaGPU;
    }
    gp_usage_input u{};
    u.n_nodes = (int32_t)N;
    u.alloc_cpu_milli = call.ac.data(); u.alloc_mem_bytes = call.am.data(); u.alloc_gpu = call.ag.data();
    u.overhead_cpu_milli = oc.data(); u.overhead_mem_bytes = om.data(); u.overhead_gpu = og.data();
    u.n_reservations = (int64_t)R; u.res_node = rn.data(); u.res_cpu_milli = rc.data(); u.res_mem_bytes = rm.data(); u.res_gpu = rg.data();
    gangpack::Device& dev = gangpack::Device::Get();
    dev.check(gp_reconcile_find_nodes(dev.ctx(), &u, &call.nd, &call.a, &call.out), "gp_reconcile_find_nodes");
    return call.Results(nodes);
}

// The overhead computer (internal/extender/overhead.go): the event side on the host, the per-call side in one
// gp_node_overhead call.  Only the fields the computer reads are kept.
struct Container { resources::Resources Requests; };  // cpu, memory and nvidia.com/gpu of Resources.Requests
struct Pod {
    std::string UID, Namespace, Name, NodeName, SchedulerName;
    std::map<std::string, std::string> Labels;
    std::vector<Container> Containers, InitContainers;
};

// podToResources (overhead.go:195-209): the containers summed, then a per-dimension max with each init container
inline resources::Resources PodToResources(const Pod& pod) {
    resources::Resources r;
    for (const Container& c : pod.Containers) r.Add(c.Requests);
    for (const Container& c : pod.InitContainers) {
        r.CPU = std::max(r.CPU, c.Requests.CPU);
        r.Memory = std::max(r.Memory, c.Requests.Memory);
        r.NvidiaGPU = std::max(r.NvidiaGPU, c.Requests.NvidiaGPU);
    }
    return r;
}

// The lister and reservation views the per-call side reads: the pod lister by (namespace, name), the ResourceReservation
// cache by (namespace, appID) with its Status.Pods values, the soft store by appID with its Reservations keys.
struct OverheadView {
    std::map<std::pair<std::string, std::string>, Pod> Pods;
    std::map<std::pair<std::string, std::string>, std::vector<std::string>> ResourceReservations;
    std::map<std::string, std::vector<std::string>> SoftReservations;
};

class OverheadComputer {
public:
    // FilteringResourceEventHandler{podHasNodeName}: an add of a bound pod, the update that binds a pod, and the update that
    // unbinds one (a delete) change the records; other updates change nothing
    void AddPod(const Pod& p) { if (!p.NodeName.empty()) record(p); }
    void UpdatePod(const Pod& oldPod, const Pod& newPod) {
        if (!newPod.NodeName.empty() && oldPod.NodeName.empty()) record(newPod);
        else if (newPod.NodeName.empty() && !oldPod.NodeName.empty()) remove(oldPod);
    }
    void DeletePod(const Pod& p) { if (!p.NodeName.empty()) remove(p); }

    resources::NodeGroupResources GetOverhead(const OverheadView& v, const std::vector<std::string>& nodes) const {
        return compute(v, nodes).first;
    }
    resources::NodeGroupResources GetNonSchedulableOverhead(const OverheadView& v, const std::vector<std::string>& nodes) const {
        return compute(v, nodes).second;
    }
    // getOverheadByNode (overhead.go:105-117): both maps from one device call; *warned = pods the reference logs a warning for
    std::pair<resources::NodeGroupResources, resources::NodeGroupResources> compute(const OverheadView& v, const std::vector<std::string>& nodes,
                                                                                    int64_t* warned = nullptr) const {
        std::map<std::string, int32_t> nodeIx, keyIx, appIx, nameIx;
        auto id = [](std::map<std::string, int32_t>& m, const std::string& s) { return m.emplace(s, (int32_t)m.size()).first->second; };
        auto key = [](const std::string& ns, const std::string& app) { return ns + '\x00' + app; };
        std::vector<int32_t> query;
        for (const auto& n : nodes) query.push_back(id(nodeIx, n));
        std::vector<int32_t> rrKey, rrName, softApp, softName;
        std::vector<int64_t> rrOff{0}, softOff{0};
        for (const auto& kv : v.ResourceReservations) {
            rrKey.push_back(id(keyIx, key(kv.first.first, kv.first.second)));
            for (const auto& s : kv.second) rrName.push_back(id(nameIx, s));
            rrOff.push_back((int64_t)rrName.size());
        }
        for (const auto& kv : v.SoftReservations) {
            softApp.push_back(id(appIx, kv.first));
            for (const auto& s : kv.second) softName.push_back(id(nameIx, s));
            softOff.push_back((int64_t)softName.size());
        }
        const size_t P = slots_.size();
        std::vector<int32_t> node(P, -1), ak(P, -1), ai(P, -1), nm(P, 0);
        std::vector<int64_t> cpu(P), mem(P), gpu(P);
        std::vector<uint8_t> listed(P), exe(P), spark(P);
        for (size_t i = 0; i < P; ++i) {
            const Slot& s = slots_[i];
            if (!s.used) continue;
            node[i] = id(nodeIx, s.node);
            cpu[i] = s.requests.CPU; mem[i] = s.requests.Memory; gpu[i] = s.requests.NvidiaGPU;
            auto it = v.Pods.find({s.ns, s.name});
            if (it == v.Pods.end()) continue;
            const Pod& pod = it->second;
            listed[i] = 1;
            auto app = pod.Labels.find("spark-app-id");
            if (app != pod.Labels.end()) { ak[i] = id(keyIx, key(pod.Namespace, app->second)); ai[i] = id(appIx, app->second); }
            nm[i] = id(nameIx, pod.Name);
            auto role = pod.Labels.find("spark-role");
            exe[i] = role != pod.Labels.end() && role->second == "executor";
            spark[i] = pod.SchedulerName == "spark-scheduler";
        }
        gp_overhead_pods in{};
        in.n_pods = (int64_t)P; in.n_node_ids = (int32_t)nodeIx.size(); in.n_app_keys = (int32_t)keyIx.size();
        in.n_app_ids = (int32_t)appIx.size(); in.n_names = (int32_t)nameIx.size();
        in.node_id = node.data(); in.req_cpu_milli = cpu.data(); in.req_mem_bytes = mem.data(); in.req_gpu = gpu.data();
        in.listed = listed.data(); in.app_key = ak.data(); in.app_id = ai.data(); in.name_id = nm.data();
        in.is_executor = exe.data(); in.spark_scheduler = spark.data();
        gp_overhead_reservations rsv{};
        rsv.n_rr = (int32_t)rrKey.size(); rsv.n_soft = (int32_t)softApp.size();
        rsv.rr_app_key = rrKey.data(); rsv.rr_pod_off = rrOff.data(); rsv.rr_pod_name = rrName.data();
        rsv.soft_app_id = softApp.data(); rsv.soft_pod_off = softOff.data(); rsv.soft_pod_name = softName.data();
        const size_t N = nodes.size();
        std::vector<int64_t> o(6 * std::max<size_t>(N, 1));
        int64_t nw = 0;
        gp_overhead_out out{o.data(), o.data() + N, o.data() + 2 * N, o.data() + 3 * N, o.data() + 4 * N, o.data() + 5 * N, nullptr, &nw};
        gangpack::Device& dev = gangpack::Device::Get();
        dev.check(gp_node_overhead(dev.ctx(), &in, &rsv, (int32_t)N, query.data(), &out), "gp_node_overhead");
        std::pair<resources::NodeGroupResources, resources::NodeGroupResources> res;
        for (size_t i = 0; i < N; ++i) {
            res.first[nodes[i]] = resources::CreateResources(o[i], o[N + i], o[2 * N + i]);
            res.second[nodes[i]] = resources::CreateResources(o[3 * N + i], o[4 * N + i], o[5 * N + i]);
        }
        if (warned) *warned = nw;
        return res;
    }

private:
    struct Slot { bool used = false; std::string ns, name, node; resources::Resources requests; };
    void record(const Pod& p) {                            // addPodRequests (overhead.go:163-174)
        auto k = std::make_pair(p.NodeName, p.UID);
        auto it = at_.find(k);
        size_t i;
        if (it != at_.end()) i = it->second;
        else if (!free_.empty()) { i = free_.back(); free_.pop_back(); at_.emplace(k, i); }
        else { i = slots_.size(); slots_.emplace_back(); at_.emplace(k, i); }
        slots_[i] = Slot{true, p.Namespace, p.Name, p.NodeName, PodToResources(p)};
    }
    void remove(const Pod& p) {                            // deletePodRequests (:176-193)
        auto it = at_.find({p.NodeName, p.UID});
        if (it == at_.end()) return;
        slots_[it->second] = Slot{};
        free_.push_back(it->second);
        at_.erase(it);
    }
    std::vector<Slot> slots_;
    std::vector<size_t> free_;
    std::map<std::pair<std::string, std::string>, size_t> at_;   // (node, UID) -> slot: the reference's ClusterRequests
};

// The overhead computer over the context's resident overhead table (gp_overhead_table_*): the pod events of
// OverheadComputer plus the pod lister's, the ResourceReservation cache's and the soft store's, as the informer handlers
// deliver them.  compute() sends what changed since the last call as at most one gp_overhead_table_update and answers with
// one gp_overhead_table_query.  Ids come from reference-counted interners, so the ids of names that are gone are reused; a
// capacity that would be exceeded is doubled and the whole state replayed after a reset.  The table belongs to the
// device context, so one instance per context.
class ResidentOverheadComputer : public gangpack::ResidentTable<gp_overhead_table_size> {
public:
    explicit ResidentOverheadComputer(gp_overhead_table_size initial = {64, 64, 64, 64, 64}) : ResidentTable(initial) {}
    ResidentOverheadComputer(const ResidentOverheadComputer&) = delete;            // rows hold pointers to its interners
    ResidentOverheadComputer& operator=(const ResidentOverheadComputer&) = delete;

    void AddPod(const Pod& p) { if (!p.NodeName.empty()) record(p); }
    void UpdatePod(const Pod& oldPod, const Pod& newPod) {
        if (!newPod.NodeName.empty() && oldPod.NodeName.empty()) record(newPod);
        else if (newPod.NodeName.empty() && !oldPod.NodeName.empty()) remove(oldPod);
    }
    void DeletePod(const Pod& p) { if (!p.NodeName.empty()) remove(p); }

    // the pod lister: the pod now at (namespace, name), or none
    void SetListerPod(const Pod& p) {
        const auto k = std::make_pair(p.Namespace, p.Name);
        lister_[k] = p;
        refreshPod(k);
    }
    void DeleteListerPod(const std::string& ns, const std::string& name) {
        if (lister_.erase({ns, name})) refreshPod({ns, name});
    }
    // the ResourceReservation (namespace, appID) with its Status.Pods values (they may repeat), and its deletion
    void SetResourceReservation(const std::string& ns, const std::string& app, const std::vector<std::string>& pods) {
        const int32_t k = keys_.acquire(appKey(ns, app));
        touchFlag(k);
        flags_.insert(k);
        hold(0, k, pods);
        dropReservation(ns, app);
        rrs_[{ns, app}] = pods;
    }
    void DeleteResourceReservation(const std::string& ns, const std::string& app) {
        if (!rrs_.count({ns, app})) return;
        const int32_t k = keys_.id.at(appKey(ns, app));
        touchFlag(k);
        flags_.erase(k);
        dropReservation(ns, app);
    }
    // the soft store's entry of appID with its Reservations keys, and its deletion
    void SetSoftReservation(const std::string& app, const std::vector<std::string>& pods) {
        hold(1, apps_.acquire(app), pods);
        dropSoft(app);
        soft_[app] = pods;
    }
    void DeleteSoftReservation(const std::string& app) { if (soft_.count(app)) dropSoft(app); }

    // For the entries that read the table in place: send the pending delta (at most one update), the table's id of each node
    // name (-1: no records, overhead zero), and a reset and replay of the whole state at the next flush (after a refusal).
    void Flush(gangpack::Device& dev) { flush(dev); }
    std::vector<int32_t> NodeIDs(const std::vector<std::string>& nodes) const {
        std::vector<int32_t> ids(nodes.size(), -1);
        for (size_t i = 0; i < nodes.size(); ++i) {
            auto it = nodes_.id.find(nodes[i]);
            if (it != nodes_.id.end()) ids[i] = it->second;
        }
        return ids;
    }

    resources::NodeGroupResources GetOverhead(const std::vector<std::string>& nodes) { return compute(nodes).first; }
    resources::NodeGroupResources GetNonSchedulableOverhead(const std::vector<std::string>& nodes) { return compute(nodes).second; }
    // getOverheadByNode (overhead.go:105-117): both maps; *warned = pods the reference logs a warning for.  A node without an
    // id has no records: it answers zero without being sent.
    std::pair<resources::NodeGroupResources, resources::NodeGroupResources> compute(const std::vector<std::string>& nodes,
                                                                                    int64_t* warned = nullptr) {
        gangpack::Device& dev = gangpack::Device::Get();
        flush(dev);
        std::vector<int32_t> query;
        std::vector<size_t> at;
        for (size_t i = 0; i < nodes.size(); ++i) {
            auto it = nodes_.id.find(nodes[i]);
            if (it != nodes_.id.end()) { query.push_back(it->second); at.push_back(i); }
        }
        const size_t Q = query.size();
        std::vector<int64_t> o(6 * std::max<size_t>(Q, 1));
        int64_t nw = 0;
        gp_overhead_out out{o.data(), o.data() + Q, o.data() + 2 * Q, o.data() + 3 * Q, o.data() + 4 * Q, o.data() + 5 * Q, nullptr, &nw};
        dev.check(gp_overhead_table_query(dev.ctx(), (int32_t)Q, query.data(), &out), "gp_overhead_table_query");
        std::pair<resources::NodeGroupResources, resources::NodeGroupResources> res;
        for (const auto& n : nodes) res.first[n] = res.second[n] = resources::Zero();
        for (size_t j = 0; j < Q; ++j) {
            res.first[nodes[at[j]]] = resources::CreateResources(o[j], o[Q + j], o[2 * Q + j]);
            res.second[nodes[at[j]]] = resources::CreateResources(o[3 * Q + j], o[4 * Q + j], o[5 * Q + j]);
        }
        if (warned) *warned = nw;
        return res;
    }

private:
    struct Ids {                                   // dense ids with reference counts
        std::unordered_map<std::string, int32_t> id;
        std::vector<int32_t> count, freed;
        int32_t acquire(const std::string& k) {
            auto it = id.find(k);
            int32_t i;
            if (it != id.end()) i = it->second;
            else {
                if (!freed.empty()) { i = freed.back(); freed.pop_back(); }
                else { i = (int32_t)count.size(); count.push_back(0); }
                id.emplace(k, i);
            }
            ++count[(size_t)i];
            return i;
        }
        void release(const std::string& k) {
            auto it = id.find(k);
            const int32_t i = it->second;
            if (--count[(size_t)i] == 0) { id.erase(it); freed.push_back(i); }
        }
        int32_t bound() const { return (int32_t)count.size(); }
    };
    struct Row {                                   // one slot's columns as the table holds them
        int32_t node = -1;
        int64_t req[3] = {0, 0, 0};
        uint8_t listed = 0;
        int32_t ak = -1, ai = -1, nm = 0;
        uint8_t exe = 0, spark = 0;
        bool operator==(const Row& o) const {
            return node == o.node && req[0] == o.req[0] && req[1] == o.req[1] && req[2] == o.req[2] && listed == o.listed &&
                   ak == o.ak && ai == o.ai && nm == o.nm && exe == o.exe && spark == o.spark;
        }
        bool operator!=(const Row& o) const { return !(*this == o); }
    };
    struct Slot { bool used = false; std::string ns, name, node; resources::Resources requests; };
    using Member = std::tuple<int, int32_t, int32_t>;   // (kind, app, name)
    using PodKey = std::pair<std::string, std::string>;

    static std::string appKey(const std::string& ns, const std::string& app) { return ns + '\x00' + app; }

    void record(const Pod& p) {                    // addPodRequests (overhead.go:163-174), the slots of OverheadComputer
        auto k = std::make_pair(p.NodeName, p.UID);
        auto it = at_.find(k);
        size_t i;
        if (it != at_.end()) i = it->second;
        else if (!free_.empty()) { i = free_.back(); free_.pop_back(); at_.emplace(k, i); }
        else { i = slots_.size(); slots_.emplace_back(); at_.emplace(k, i); }
        slots_[i] = Slot{true, p.Namespace, p.Name, p.NodeName, PodToResources(p)};
        refresh(i);
    }
    void remove(const Pod& p) {                    // deletePodRequests (:176-193)
        auto it = at_.find({p.NodeName, p.UID});
        if (it == at_.end()) return;
        const size_t i = it->second;
        slots_[i] = Slot{};
        free_.push_back(i);
        at_.erase(it);
        refresh(i);
    }
    void refreshPod(const PodKey& k) {
        auto it = byPod_.find(k);
        if (it == byPod_.end()) return;
        const std::vector<size_t> at(it->second.begin(), it->second.end());
        for (size_t i : at) refresh(i);
    }
    // the slot's row from its record and the lister's current pod; the references of the new row are taken before the old
    // row's are released
    void refresh(size_t i) {
        if (rows_.size() < slots_.size()) { rows_.resize(slots_.size()); refs_.resize(slots_.size()); podOf_.resize(slots_.size()); }
        const Slot& s = slots_[i];
        Row r;
        std::vector<std::pair<Ids*, std::string>> refs;
        auto take = [&](Ids& ids, const std::string& k) { refs.emplace_back(&ids, k); return ids.acquire(k); };
        if (s.used) {
            r.node = take(nodes_, s.node);
            r.req[0] = s.requests.CPU; r.req[1] = s.requests.Memory; r.req[2] = s.requests.NvidiaGPU;
            auto it = lister_.find({s.ns, s.name});
            if (it != lister_.end()) {
                const Pod& pod = it->second;
                r.listed = 1;
                auto app = pod.Labels.find("spark-app-id");
                if (app != pod.Labels.end()) { r.ak = take(keys_, appKey(pod.Namespace, app->second)); r.ai = take(apps_, app->second); }
                r.nm = take(names_, pod.Name);
                auto role = pod.Labels.find("spark-role");
                r.exe = role != pod.Labels.end() && role->second == "executor";
                r.spark = pod.SchedulerName == "spark-scheduler";
            }
        }
        for (auto& ref : refs_[i]) ref.first->release(ref.second);
        dirty_.emplace(i, rows_[i]);
        rows_[i] = r;
        refs_[i] = std::move(refs);
        const PodKey now = s.used ? PodKey{s.ns, s.name} : PodKey{};
        if (podOf_[i] != now) {
            if (!podOf_[i].second.empty() || !podOf_[i].first.empty()) {
                auto& set = byPod_[podOf_[i]];
                set.erase(i);
                if (set.empty()) byPod_.erase(podOf_[i]);
            }
            if (s.used) byPod_[now].insert(i);
            podOf_[i] = now;
        }
    }
    void touchFlag(int32_t k) { flagTouched_.emplace(k, flags_.count(k) > 0); }
    // one holder of (kind, app, name) per distinct name; each holds a reference on the name's id
    void hold(int kind, int32_t app, const std::vector<std::string>& pods) {
        for (const auto& n : std::set<std::string>(pods.begin(), pods.end())) {
            const Member m{kind, app, names_.acquire(n)};
            int32_t& c = members_[m];
            memberTouched_.emplace(m, c > 0);
            ++c;
        }
    }
    void release(int kind, int32_t app, const std::vector<std::string>& pods) {
        for (const auto& n : std::set<std::string>(pods.begin(), pods.end())) {
            const Member m{kind, app, names_.id.at(n)};
            auto it = members_.find(m);
            memberTouched_.emplace(m, it->second > 0);
            if (--it->second == 0) members_.erase(it);
            names_.release(n);
        }
    }
    void dropReservation(const std::string& ns, const std::string& app) {
        auto it = rrs_.find({ns, app});
        if (it == rrs_.end()) return;
        release(0, keys_.id.at(appKey(ns, app)), it->second);
        keys_.release(appKey(ns, app));
        rrs_.erase(it);
    }
    void dropSoft(const std::string& app) {
        auto it = soft_.find(app);
        if (it == soft_.end()) return;
        release(1, apps_.id.at(app), it->second);
        apps_.release(app);
        soft_.erase(it);
    }

    // The changes since the last update (everything after a reset) as one gp_overhead_table_update
    void flush(gangpack::Device& dev) {
        Grow(size_.n_slots, (int64_t)slots_.size());
        Grow(size_.n_node_ids, nodes_.bound()); Grow(size_.n_app_keys, keys_.bound()); Grow(size_.n_app_ids, apps_.bound());
        Grow(size_.n_names, names_.bound());
        std::vector<int32_t> slot, node, ak, ai, nm, rrKey, mApp, mName;
        std::vector<int64_t> cpu, mem, gpu;
        std::vector<uint8_t> listed, exe, spark, rrOn, mKind, mPresent;
        auto row = [&](size_t i) {
            const Row& r = rows_[i];
            slot.push_back((int32_t)i); node.push_back(r.node);
            cpu.push_back(r.req[0]); mem.push_back(r.req[1]); gpu.push_back(r.req[2]);
            listed.push_back(r.listed); ak.push_back(r.ak); ai.push_back(r.ai); nm.push_back(r.nm);
            exe.push_back(r.exe); spark.push_back(r.spark);
        };
        auto member = [&](const Member& m, bool present) {
            mKind.push_back((uint8_t)std::get<0>(m)); mApp.push_back(std::get<1>(m)); mName.push_back(std::get<2>(m));
            mPresent.push_back(present);
        };
        if (Replaying()) {
            for (size_t i = 0; i < rows_.size(); ++i) if (rows_[i] != Row{}) row(i);
            for (int32_t k : flags_) { rrKey.push_back(k); rrOn.push_back(1); }
            for (const auto& kv : members_) member(kv.first, true);
        } else {
            for (const auto& kv : dirty_) if (rows_[kv.first] != kv.second) row(kv.first);
            for (const auto& kv : flagTouched_) {
                const bool on = flags_.count(kv.first) > 0;
                if (on != kv.second) { rrKey.push_back(kv.first); rrOn.push_back(on); }
            }
            for (const auto& kv : memberTouched_) {
                auto it = members_.find(kv.first);
                const bool on = it != members_.end() && it->second > 0;
                if (on != kv.second) member(kv.first, on);
            }
        }
        gp_overhead_delta d{};
        d.n_write = (int64_t)slot.size();
        d.slot = slot.data(); d.node_id = node.data(); d.req_cpu_milli = cpu.data(); d.req_mem_bytes = mem.data(); d.req_gpu = gpu.data();
        d.listed = listed.data(); d.app_key = ak.data(); d.app_id = ai.data(); d.name_id = nm.data();
        d.is_executor = exe.data(); d.spark_scheduler = spark.data();
        d.n_rr = (int32_t)rrKey.size(); d.rr_app_key = rrKey.data(); d.rr_exists = rrOn.data();
        d.n_member = (int64_t)mKind.size();
        d.member_kind = mKind.data(); d.member_app = mApp.data(); d.member_name = mName.data(); d.member_present = mPresent.data();
        Send(dev, gp_overhead_table_reset, "gp_overhead_table_reset", gp_overhead_table_update, "gp_overhead_table_update",
             slot.empty() && rrKey.empty() && mKind.empty() ? nullptr : &d);
        dirty_.clear(); flagTouched_.clear(); memberTouched_.clear();
    }

    std::vector<Slot> slots_;
    std::vector<size_t> free_;
    std::map<std::pair<std::string, std::string>, size_t> at_;   // (node, UID) -> slot
    std::vector<Row> rows_;
    std::vector<std::vector<std::pair<Ids*, std::string>>> refs_;
    std::vector<PodKey> podOf_;
    std::map<PodKey, std::set<size_t>> byPod_;                    // (namespace, name) -> slots whose record names that pod
    Ids nodes_, keys_, apps_, names_;
    std::map<PodKey, Pod> lister_;
    std::map<PodKey, std::vector<std::string>> rrs_;
    std::map<std::string, std::vector<std::string>> soft_;
    std::set<int32_t> flags_;
    std::map<Member, int32_t> members_;
    std::map<size_t, Row> dirty_;                                 // -> the row the table holds
    std::map<int32_t, bool> flagTouched_;
    std::map<Member, bool> memberTouched_;
};

// GetReservedResources' rows (resourcereservations.go:258-263) over the context's resident reservation table
// (gp_reservation_table_*): the ResourceReservation cache's and the soft store's events as their handlers deliver them, one
// slot per Spec.Reservations entry or soft reservation.  Flush() sends what changed since the last one as at most one
// gp_reservation_table_update -- call it once per Predicate, before gp_prepare_cluster_*_resident or
// gp_reschedule_from_reservations_resident with NodeIDs(nodes).  Freed slots are reused and node ids are reference-counted;
// a capacity that would be exceeded is doubled, and after a reset, a refused or a failed update the whole state is sent
// again until an update succeeds.  The table belongs to the device context, so one instance per context.
class ResidentReservations : public gangpack::ResidentTable<gp_reservation_table_size> {
public:
    struct Reservation { std::string Node; resources::Resources Res; };
    using Entries = std::map<std::string, Reservation>;           // name (reservation entry or pod) -> reservation

    explicit ResidentReservations(gp_reservation_table_size initial = {64, 64}) : ResidentTable(initial) {}

    // a ResourceReservation created, updated or rewritten by compaction (its Spec.Reservations), and its deletion
    void SetResourceReservation(const std::string& ns, const std::string& app, const Entries& e) { set(0, ns + '\x00' + app, e, rrs_); }
    void DeleteResourceReservation(const std::string& ns, const std::string& app) { set(0, ns + '\x00' + app, {}, rrs_); }
    // the soft store's reservations of appID (pod name -> reservation), and their removal
    void SetSoftReservations(const std::string& app, const Entries& e) { set(1, app, e, soft_); }
    void DeleteSoftReservations(const std::string& app) { set(1, app, {}, soft_); }

    // the table's id of each node name, -1 for a node no reservation names
    std::vector<int32_t> NodeIDs(const std::vector<std::string>& nodes) const {
        std::vector<int32_t> ids(nodes.size(), -1);
        for (size_t i = 0; i < nodes.size(); ++i) {
            auto it = nodes_.find(nodes[i]);
            if (it != nodes_.end()) ids[i] = it->second;
        }
        return ids;
    }

    // GetReservedResources' rows as the per-call reconciler takes them
    std::vector<ReconcileRow> Rows() const {
        std::vector<ReconcileRow> rows;
        for (const auto* store : {&rrs_, &soft_})
            for (const auto& owner : *store)
                for (const auto& e : owner.second) rows.push_back(ReconcileRow{e.second.Node, e.second.Res});
        return rows;
    }

    void Flush(gangpack::Device& dev) {
        Grow(size_.n_slots, (int64_t)rows_.size());
        Grow(size_.n_node_ids, (int64_t)nodeCount_.size());
        std::vector<int32_t> slot, node;
        std::vector<int64_t> cpu, mem, gpu;
        auto row = [&](size_t i) {
            slot.push_back((int32_t)i); node.push_back(rows_[i].node);
            cpu.push_back(rows_[i].v[0]); mem.push_back(rows_[i].v[1]); gpu.push_back(rows_[i].v[2]);
        };
        if (Replaying()) {
            for (size_t i = 0; i < rows_.size(); ++i) if (rows_[i].node != -1) row(i);
        } else {
            for (const auto& kv : dirty_) if (rows_[kv.first] != kv.second) row(kv.first);
        }
        gp_reservation_delta d{(int64_t)slot.size(), slot.data(), node.data(), cpu.data(), mem.data(), gpu.data()};
        Send(dev, gp_reservation_table_reset, "gp_reservation_table_reset", gp_reservation_table_update, "gp_reservation_table_update",
             slot.empty() ? nullptr : &d);
        dirty_.clear();
    }

private:
    struct Row {
        int32_t node = -1;
        int64_t v[3] = {0, 0, 0};
        bool operator!=(const Row& o) const { return node != o.node || v[0] != o.v[0] || v[1] != o.v[1] || v[2] != o.v[2]; }
    };
    using Key = std::tuple<int, std::string, std::string>;       // (kind, owner, name)

    void set(int kind, const std::string& owner, const Entries& now, std::map<std::string, Entries>& store) {
        Entries old;
        auto it = store.find(owner);
        if (it != store.end()) { old = std::move(it->second); store.erase(it); }
        if (!now.empty()) store[owner] = now;
        for (const auto& kv : old)
            if (!now.count(kv.first)) {
                auto s = slot_.find(Key{kind, owner, kv.first});
                write(s->second, nullptr);
                slot_.erase(s);
            }
        for (const auto& kv : now) {
            const Key k{kind, owner, kv.first};
            auto s = slot_.find(k);
            size_t at;
            if (s == slot_.end()) {
                if (!free_.empty()) { at = free_.back(); free_.pop_back(); }
                else { at = rows_.size(); rows_.emplace_back(); nodeOf_.emplace_back(); }
                slot_.emplace(k, at);
            } else {
                at = s->second;
                auto o = old.find(kv.first);
                if (o != old.end() && o->second.Node == kv.second.Node && o->second.Res.Eq(kv.second.Res)) continue;
            }
            write(at, &kv.second);
        }
    }
    // slot at := r, or free it (r NULL); the node reference of the new row is taken before the old row's is released
    void write(size_t at, const Reservation* r) {
        dirty_.emplace(at, rows_[at]);
        Row row;
        if (r) {
            row.node = acquire(r->Node);
            row.v[0] = r->Res.CPU; row.v[1] = r->Res.Memory; row.v[2] = r->Res.NvidiaGPU;
        }
        if (!nodeOf_[at].empty()) release(nodeOf_[at]);
        rows_[at] = row;
        nodeOf_[at] = r ? r->Node : std::string();
        if (!r) free_.push_back(at);
    }
    int32_t acquire(const std::string& n) {
        auto it = nodes_.find(n);
        int32_t i;
        if (it != nodes_.end()) i = it->second;
        else {
            if (!freeIds_.empty()) { i = freeIds_.back(); freeIds_.pop_back(); }
            else { i = (int32_t)nodeCount_.size(); nodeCount_.push_back(0); }
            nodes_.emplace(n, i);
        }
        ++nodeCount_[(size_t)i];
        return i;
    }
    void release(const std::string& n) {
        auto it = nodes_.find(n);
        const int32_t i = it->second;
        if (--nodeCount_[(size_t)i] == 0) { nodes_.erase(it); freeIds_.push_back(i); }
    }

    std::map<std::string, Entries> rrs_, soft_;
    std::map<Key, size_t> slot_;
    std::vector<Row> rows_;
    std::vector<std::string> nodeOf_;                             // per slot: the node name its row holds ("" = free)
    std::vector<size_t> free_;
    std::unordered_map<std::string, int32_t> nodes_;
    std::vector<int32_t> nodeCount_, freeIds_;
    std::map<size_t, Row> dirty_;                                 // -> the row the table holds
};

// ReconcileFindNodes over the resident tables (gp_reconcile_find_nodes_resident): each table's pending delta is flushed once,
// then one device call reads every reservation and GetOverhead in place.  A refused call resets and replays both tables and
// is made again per call, over Rows() and GetOverhead, which answers or refuses as the per-call entry does.
inline std::vector<ReconcileResult> ReconcileFindNodesResident(const std::vector<ReconcileNode>& nodes, ResidentReservations& reservations,
                                                               ResidentOverheadComputer& overhead, const std::string& instanceGroupLabel,
                                                               const std::vector<StaleDriver>& drivers) {
    gangpack::Device& dev = gangpack::Device::Get();
    reservations.Flush(dev);
    overhead.Flush(dev);
    std::vector<std::string> names;
    for (const auto& n : nodes) names.push_back(n.Name);
    const std::vector<int32_t> ids = reservations.NodeIDs(names), oids = overhead.NodeIDs(names);
    ReconcileCall call(nodes, instanceGroupLabel, drivers);
    gp_resident_usage u{};
    u.n_nodes = (int32_t)nodes.size(); u.node_id = ids.data();
    u.alloc_cpu_milli = call.ac.data(); u.alloc_mem_bytes = call.am.data(); u.alloc_gpu = call.ag.data();
    u.overhead_node_id = oids.data();
    if (gp_reconcile_find_nodes_resident(dev.ctx(), &u, &call.nd, &call.a, &call.out) == GP_OK) return call.Results(nodes);
    reservations.Replay();
    overhead.Replay();
    reservations.Flush(dev);
    return ReconcileFindNodes(nodes, reservations.Rows(), overhead.GetOverhead(names), instanceGroupLabel, drivers);
}

inline std::vector<bool> UnschedulablePodMarker::DoesPodsExceedClusterCapacity(const std::vector<CapacityNode>& nodes,
                                                                               ResidentOverheadComputer& overhead,
                                                                               const std::unordered_map<std::string, int32_t>& nodeClass,
                                                                               int32_t nClasses, const std::vector<StaleDriver>& drivers) const {
    gangpack::Device& dev = gangpack::Device::Get();
    overhead.Flush(dev);
    const size_t N = nodes.size(), Q = drivers.size();
    std::vector<std::string> names;
    std::vector<int64_t> ac(N + 1), am(N + 1), ag(N + 1);
    std::vector<int32_t> zone(N + 1), group(N + 1);
    std::unordered_map<std::string, int32_t> zoneId;
    for (size_t i = 0; i < N; ++i) {
        names.push_back(nodes[i].Name);
        ac[i] = nodes[i].Allocatable.CPU; am[i] = nodes[i].Allocatable.Memory; ag[i] = nodes[i].Allocatable.NvidiaGPU;
        zone[i] = zoneId.emplace(nodes[i].ZoneLabel, (int32_t)zoneId.size()).first->second;
        auto c = nodeClass.find(nodes[i].Name);
        group[i] = c == nodeClass.end() ? -1 : c->second;
    }
    const std::vector<int32_t> oids = overhead.NodeIDs(names);
    std::vector<int64_t> q[6];
    std::vector<int32_t> count(Q + 1), cls(Q + 1);
    for (auto& col : q) col.resize(Q + 1);
    for (size_t i = 0; i < Q; ++i) {
        const StaleDriver& d = drivers[i];
        q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
        q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
        count[i] = d.MinExecutorCount; cls[i] = d.AffinityClass;
    }
    gp_capacity_nodes n{};
    n.n_nodes = (int32_t)N;
    n.alloc_cpu_milli = ac.data(); n.alloc_mem_bytes = am.data(); n.alloc_gpu = ag.data();
    n.n_zones = std::max<int32_t>(1, (int32_t)zoneId.size()); n.zone_id = zone.data();
    n.n_groups = std::max<int32_t>(1, nClasses); n.node_group = group.data();
    gp_apps a{};
    a.n_apps = (int32_t)Q;
    a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
    a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
    a.exe_count = count.data(); a.group = cls.data();
    std::vector<uint8_t> out(Q + 1);
    if (gp_exceeds_cluster_capacity_resident(dev.ctx(), &n, oids.data(), &a, Packer(), out.data()) == GP_OK)
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    overhead.Replay();
    const resources::NodeGroupResources nonsched = overhead.GetNonSchedulableOverhead(names);
    resources::NodeGroupSchedulingMetadata md;
    for (const auto& node : nodes) {
        resources::NodeSchedulingMetadata m;
        m.SchedulableResources = node.Allocatable;
        m.SchedulableResources.Sub(nonsched.at(node.Name));
        m.ZoneLabel = node.ZoneLabel;
        md[node.Name] = m;
    }
    return DoesPodsExceedClusterCapacity(md, nodeClass, nClasses, drivers);
}

inline std::vector<bool> UnschedulablePodMarker::DoesPodsExceedClusterCapacity(const std::vector<CapacityNode>& nodes,
                                                                               ResidentOverheadComputer& overhead,
                                                                               affinity::ResidentLabels& labels,
                                                                               const std::vector<affinity::Program>& programs,
                                                                               const std::vector<AffinityStaleDriver>& drivers,
                                                                               std::vector<bool>* affinityError) const {
    gangpack::Device& dev = gangpack::Device::Get();
    overhead.Flush(dev);
    labels.Flush(dev);
    const size_t N = nodes.size(), Q = drivers.size();
    std::vector<std::string> names;
    std::vector<int64_t> ac(N + 1), am(N + 1), ag(N + 1);
    std::vector<int32_t> zone(N + 1);
    std::unordered_map<std::string, int32_t> zoneId;
    for (size_t i = 0; i < N; ++i) {
        names.push_back(nodes[i].Name);
        ac[i] = nodes[i].Allocatable.CPU; am[i] = nodes[i].Allocatable.Memory; ag[i] = nodes[i].Allocatable.NvidiaGPU;
        zone[i] = zoneId.emplace(nodes[i].ZoneLabel, (int32_t)zoneId.size()).first->second;
    }
    const std::vector<int32_t> oids = overhead.NodeIDs(names), lids = labels.NodeIDs(names);
    std::vector<int64_t> q[6];
    std::vector<int32_t> count(Q + 1), prog(Q + 1);
    for (auto& col : q) col.resize(Q + 1);
    for (size_t i = 0; i < Q; ++i) {
        const AffinityStaleDriver& d = drivers[i];
        q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
        q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
        count[i] = d.MinExecutorCount; prog[i] = d.Affinity;
    }
    const affinity::Encoded e = labels.EncodePrograms(names, programs);
    const gp_node_affinities p = e.Programs();
    const gp_resident_labels rl{(int32_t)N, 0, lids.data()};
    gp_capacity_nodes n{};
    n.n_nodes = (int32_t)N;
    n.alloc_cpu_milli = ac.data(); n.alloc_mem_bytes = am.data(); n.alloc_gpu = ag.data();
    n.n_zones = std::max<int32_t>(1, (int32_t)zoneId.size()); n.zone_id = zone.data();
    gp_apps a{};
    a.n_apps = (int32_t)Q;
    a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
    a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
    a.exe_count = count.data(); a.group = prog.data();
    std::vector<uint8_t> out(Q + 1), err(Q + 1);
    if (gp_exceeds_cluster_capacity_affinity_label_table(dev.ctx(), &n, oids.data(), &rl, &p, &a, Packer(), out.data(), err.data()) == GP_OK) {
        if (affinityError) affinityError->assign(err.begin(), err.begin() + (std::ptrdiff_t)Q);
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    }
    overhead.Replay();
    labels.Replay();
    labels.Flush(dev);
    const resources::NodeGroupResources nonsched = overhead.GetNonSchedulableOverhead(names);
    resources::NodeGroupSchedulingMetadata md;
    for (const auto& node : nodes) {
        resources::NodeSchedulingMetadata m;
        m.SchedulableResources = node.Allocatable;
        m.SchedulableResources.Sub(nonsched.at(node.Name));
        m.ZoneLabel = node.ZoneLabel;
        md[node.Name] = m;
    }
    return DoesPodsExceedClusterCapacity(md, labels.Nodes(names), programs, drivers, affinityError);
}

// The CapacityNode list of the resident sweeps, decoded on the host from the node and label tables' own state
inline std::vector<UnschedulablePodMarker::CapacityNode> CapacityNodesOf(const std::vector<std::string>& names,
                                                                         const resources::ResidentNodes& nodes,
                                                                         const affinity::ResidentLabels& labels) {
    const resources::ResidentNodes::Columns c = nodes.PerCall(names);
    const std::vector<affinity::Node> lab = labels.Nodes(names);
    std::vector<UnschedulablePodMarker::CapacityNode> out(names.size());
    for (size_t i = 0; i < names.size(); ++i) {
        out[i].Name = names[i];
        out[i].Allocatable = resources::Resources{c.alloc[0][i], c.alloc[1][i], c.alloc[2][i]};
        auto z = lab[i].Labels.find(resources::NodeTableLabels::kZoneLabel);
        if (z != lab[i].Labels.end()) out[i].ZoneLabel = z->second;
    }
    return out;
}

// The gp_node_table_nodes of a node-table marker sweep over these names (flushed tables; the zone arguments from z)
struct MarkerNodeTable {
    std::vector<int32_t> ids, oids;
    gp_node_table_nodes nd{};
    MarkerNodeTable(const std::vector<std::string>& names, const resources::ResidentNodes& nodes, ResidentOverheadComputer& overhead,
                    const resources::NodeTableLabels& z)
        : ids(nodes.NodeIDs(names)), oids(overhead.NodeIDs(names)) {
        z.Fill(&nd);
        nd.n_nodes = (int32_t)names.size();
        nd.node_table_id = ids.data();
        nd.overhead_node_id = oids.data();
    }
};

inline std::vector<bool> UnschedulablePodMarker::DoesPodsExceedClusterCapacity(const std::vector<std::string>& names,
                                                                               resources::ResidentNodes& nodes,
                                                                               affinity::ResidentLabels& labels,
                                                                               ResidentOverheadComputer& overhead,
                                                                               const std::vector<std::string>& zones,
                                                                               const std::unordered_map<std::string, int32_t>& nodeClass,
                                                                               int32_t nClasses, const std::vector<StaleDriver>& drivers) const {
    gangpack::Device& dev = gangpack::Device::Get();
    overhead.Flush(dev);
    labels.Flush(dev);
    nodes.Flush(dev);
    const size_t N = names.size(), Q = drivers.size();
    const resources::NodeTableLabels z(labels, zones, "", {});
    MarkerNodeTable t(names, nodes, overhead, z);
    std::vector<int32_t> group(N + 1);
    for (size_t i = 0; i < N; ++i) {
        auto c = nodeClass.find(names[i]);
        group[i] = c == nodeClass.end() ? -1 : c->second;
    }
    std::vector<int64_t> q[6];
    std::vector<int32_t> count(Q + 1), cls(Q + 1);
    for (auto& col : q) col.resize(Q + 1);
    for (size_t i = 0; i < Q; ++i) {
        const StaleDriver& d = drivers[i];
        q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
        q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
        count[i] = d.MinExecutorCount; cls[i] = d.AffinityClass;
    }
    gp_apps a{};
    a.n_apps = (int32_t)Q;
    a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
    a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
    a.exe_count = count.data(); a.group = cls.data();
    std::vector<uint8_t> out(Q + 1);
    if (gp_exceeds_cluster_capacity_node_table(dev.ctx(), &t.nd, group.data(), std::max<int32_t>(1, nClasses), &a, Packer(), out.data()) == GP_OK)
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    overhead.Replay();
    labels.Replay();
    nodes.Replay();
    labels.Flush(dev);
    nodes.Flush(dev);
    return DoesPodsExceedClusterCapacity(CapacityNodesOf(names, nodes, labels), overhead, nodeClass, nClasses, drivers);
}

inline std::vector<bool> UnschedulablePodMarker::DoesPodsExceedClusterCapacity(const std::vector<std::string>& names,
                                                                               resources::ResidentNodes& nodes,
                                                                               affinity::ResidentLabels& labels,
                                                                               ResidentOverheadComputer& overhead,
                                                                               const std::vector<std::string>& zones,
                                                                               const std::vector<affinity::Program>& programs,
                                                                               const std::vector<AffinityStaleDriver>& drivers,
                                                                               std::vector<bool>* affinityError) const {
    gangpack::Device& dev = gangpack::Device::Get();
    overhead.Flush(dev);
    labels.Flush(dev);
    nodes.Flush(dev);
    const size_t Q = drivers.size();
    const resources::NodeTableLabels z(labels, zones, "", {});
    MarkerNodeTable t(names, nodes, overhead, z);
    std::vector<int64_t> q[6];
    std::vector<int32_t> count(Q + 1), prog(Q + 1);
    for (auto& col : q) col.resize(Q + 1);
    for (size_t i = 0; i < Q; ++i) {
        const AffinityStaleDriver& d = drivers[i];
        q[0][i] = d.DriverResources.CPU; q[1][i] = d.DriverResources.Memory; q[2][i] = d.DriverResources.NvidiaGPU;
        q[3][i] = d.ExecutorResources.CPU; q[4][i] = d.ExecutorResources.Memory; q[5][i] = d.ExecutorResources.NvidiaGPU;
        count[i] = d.MinExecutorCount; prog[i] = d.Affinity;
    }
    const affinity::Encoded e = labels.EncodePrograms(names, programs);
    const gp_node_affinities p = e.Programs();
    gp_apps a{};
    a.n_apps = (int32_t)Q;
    a.drv_cpu_milli = q[0].data(); a.drv_mem_bytes = q[1].data(); a.drv_gpu = q[2].data();
    a.exe_cpu_milli = q[3].data(); a.exe_mem_bytes = q[4].data(); a.exe_gpu = q[5].data();
    a.exe_count = count.data(); a.group = prog.data();
    std::vector<uint8_t> out(Q + 1), err(Q + 1);
    if (gp_exceeds_cluster_capacity_affinity_node_table(dev.ctx(), &t.nd, &p, &a, Packer(), out.data(), err.data()) == GP_OK) {
        if (affinityError) affinityError->assign(err.begin(), err.begin() + (std::ptrdiff_t)Q);
        return std::vector<bool>(out.begin(), out.begin() + (std::ptrdiff_t)Q);
    }
    overhead.Replay();
    labels.Replay();
    nodes.Replay();
    nodes.Flush(dev);
    return DoesPodsExceedClusterCapacity(CapacityNodesOf(names, nodes, labels), overhead, labels, programs, drivers, affinityError);
}

// ReconcileFindNodes over the four resident tables (gp_reconcile_find_nodes_node_table): names lists the lister's nodes (their
// order is the tie order among equal creation times); instanceGroups the values of instanceGroupLabel in group order -- ""
// (the group of a node without the label) and any driver's group not listed are appended.  Each table's pending delta is
// flushed once, then one device call reads allocatable, flags, creation, the instance-group label, every reservation and
// GetOverhead in place.  A refused call (a node whose instance group is not listed, for one) resets and replays the label
// and node tables and makes ReconcileFindNodesResident over the columns the host decodes from them.  That costs a full
// resend of both tables on every call while such a node exists: list every value the nodes carry for the key, not only
// the groups Spark manages.
inline std::vector<ReconcileResult> ReconcileFindNodesNodeTable(const std::vector<std::string>& names, resources::ResidentNodes& nodes,
                                                                affinity::ResidentLabels& labels, ResidentReservations& reservations,
                                                                ResidentOverheadComputer& overhead, const std::string& instanceGroupLabel,
                                                                const std::vector<std::string>& instanceGroups,
                                                                const std::vector<StaleDriver>& drivers) {
    gangpack::Device& dev = gangpack::Device::Get();
    labels.Flush(dev);
    nodes.Flush(dev);
    reservations.Flush(dev);
    overhead.Flush(dev);
    // every group id the call uses: the listed values, "", then the drivers' groups not listed (no node of the listed ones
    // is in them; a value id no row holds, or the value's own id when some node carries it after all).  The value list
    // and n_groups are the same list, so the gather reads exactly n_groups values.
    std::vector<std::string> groups = instanceGroups;
    if (std::find(groups.begin(), groups.end(), std::string()) == groups.end()) groups.push_back(std::string());
    const int32_t missing = (int32_t)(std::find(groups.begin(), groups.end(), std::string()) - groups.begin());
    for (const auto& d : drivers)
        if (std::find(groups.begin(), groups.end(), d.InstanceGroup) == groups.end()) groups.push_back(d.InstanceGroup);
    ReconcileCall call({}, instanceGroupLabel, drivers, &groups);
    const resources::NodeTableLabels ig(labels, {}, instanceGroupLabel, groups);
    const std::vector<int32_t> ids = nodes.NodeIDs(names), rids = reservations.NodeIDs(names), oids = overhead.NodeIDs(names);
    gp_node_table_nodes nd{};
    ig.Fill(&nd);
    nd.zone_key = -1; nd.n_zones = 1; nd.zone_value = nullptr; nd.zone_missing = -1;
    nd.driver_rank_key = -1; nd.executor_rank_key = -1;
    nd.n_nodes = (int32_t)names.size();
    nd.node_table_id = ids.data(); nd.reservation_id = rids.data(); nd.overhead_node_id = oids.data();
    if (gp_reconcile_find_nodes_node_table(dev.ctx(), &nd, (int32_t)groups.size(), missing, &call.a, &call.out) == GP_OK)
        return call.Results(names);
    labels.Replay();
    nodes.Replay();
    labels.Flush(dev);
    nodes.Flush(dev);
    const resources::ResidentNodes::Columns c = nodes.PerCall(names);
    const std::vector<affinity::Node> lab = labels.Nodes(names);
    std::vector<ReconcileNode> rn(names.size());
    for (size_t i = 0; i < names.size(); ++i) {
        rn[i].Name = names[i];
        rn[i].Allocatable = resources::Resources{c.alloc[0][i], c.alloc[1][i], c.alloc[2][i]};
        rn[i].Labels.insert(lab[i].Labels.begin(), lab[i].Labels.end());
        rn[i].Unschedulable = c.unschedulable[i] != 0;
        rn[i].Ready = c.ready[i] != 0;
        rn[i].CreationUnixNano = c.creation[i];
    }
    return ReconcileFindNodesResident(rn, reservations, overhead, instanceGroupLabel, drivers);
}

// ---- the resident driver table (gp_driver_table_*) ------------------------------------------------------------------------

// Every pending driver as the resident driver table keeps it, from the pod informer: SetDriver for a driver pod's add and
// update events (a bound or terminating pod, or one whose annotations do not parse, is deleted: resource.go:232-237),
// DeleteDriver for its delete.  Slots freed by a delete are reused, lowest first; scheduler names and instance groups are
// interned into dense ids (no instance group: -1).  Flush sends the slots that differ from what the device holds as one
// gp_driver_table_update, after a reset with doubled capacities and the whole state when a slot, group or scheduler id would
// not fit (or after Replay, or a failed flush).  The host keeps every row, so a refused device call can fall back to
// FilterToEarliestAndSort and the per-call FIFO batch over the same drivers (Pods, Pending).
class ResidentDrivers : public gangpack::ResidentTable<gp_driver_table_size> {
public:
    explicit ResidentDrivers(gp_driver_table_size size = gp_driver_table_size{64, 4, 2, 0}) : ResidentTable(size) {}

    void SetDriver(const QueuedDriverPod& pod, const std::map<std::string, std::string>& annotations) {
        ParsedSparkResources r;
        if (!pod.NodeName.empty() || pod.Deleting || !SparkResources(annotations, &r).empty()) {
            DeleteDriver(pod.UID);
            return;
        }
        Row row;
        row.present = true;
        row.creation = pod.CreationSeconds * 1000000000LL;
        row.scheduler = intern(schedulers_, pod.SchedulerName);
        row.group = pod.HasInstanceGroup ? intern(groups_, pod.InstanceGroup) : -1;
        const int64_t q[6] = {r.DriverCPUMilli, r.DriverMemoryBytes, r.DriverNvidiaGPUs, r.ExecutorCPUMilli, r.ExecutorMemoryBytes,
                              r.ExecutorNvidiaGPUs};
        for (int k = 0; k < 6; ++k) row.q[k] = q[k];
        row.count = (int32_t)r.MinExecutorCount;
        row.exact = r.Exact;
        row.affinity = acquire(pod.Affinity);
        auto it = held_.find(pod.UID);
        if (it != held_.end()) release(it->second.row.affinity);
        if (it != held_.end() && it->second.row == row && it->second.pod.CreationSeconds == pod.CreationSeconds) {
            it->second.pod.Affinity = pod.Affinity;
            return;
        }
        int32_t slot;
        if (it != held_.end()) slot = it->second.slot;
        else if (!free_.empty()) { slot = *free_.begin(); free_.erase(free_.begin()); }
        else slot = next_++;
        held_[pod.UID] = Held{slot, row, pod, r};
        uidAt_[slot] = pod.UID;
        dirty_.insert(slot);
    }
    void DeleteDriver(const std::string& uid) {
        auto it = held_.find(uid);
        if (it == held_.end()) return;
        release(it->second.row.affinity);
        dirty_.insert(it->second.slot);
        free_.insert(it->second.slot);
        uidAt_.erase(it->second.slot);
        held_.erase(it);
    }

    int32_t Slot(const std::string& uid) const { auto it = held_.find(uid); return it == held_.end() ? -1 : it->second.slot; }
    bool Holds(const std::string& uid) const { return held_.count(uid) != 0; }
    const gp_driver_table_size& Size() const { return size_; }
    // enforce_after_ns of every group id: its instance group's override, else the default (DefaultEnforceAfterPodAge)
    std::vector<int64_t> GroupAges(int64_t defaultNs, const std::map<std::string, int64_t>& overrides = {}) const {
        std::vector<int64_t> ages((size_t)size_.n_groups, defaultNs);
        for (const auto& g : groups_) {
            auto o = overrides.find(g.first);
            if (o != overrides.end()) ages[(size_t)g.second] = o->second;
        }
        return ages;
    }
    // the pending drivers as a lister lists them (slot order), and what fitEarlierDrivers reads off one of them
    std::vector<QueuedDriverPod> Pods() const {
        std::vector<QueuedDriverPod> out;
        for (const auto& kv : uidAt_) out.push_back(held_.at(kv.second).pod);
        return out;
    }
    PendingDriver Pending(const std::string& uid, bool skipIfNoFit) const {
        const Held& h = held_.at(uid);
        PendingDriver d;
        d.Name = uid;
        d.SkipIfNoFit = skipIfNoFit;
        d.Resources.DriverResources = resources::CreateResources(h.parsed.DriverCPUMilli, h.parsed.DriverMemoryBytes, h.parsed.DriverNvidiaGPUs);
        d.Resources.ExecutorResources = resources::CreateResources(h.parsed.ExecutorCPUMilli, h.parsed.ExecutorMemoryBytes, h.parsed.ExecutorNvidiaGPUs);
        d.Resources.MinExecutorCount = (int)h.parsed.MinExecutorCount;
        d.Resources.MaxExecutorCount = (int)h.parsed.MaxExecutorCount;
        return d;
    }
    bool Exact(const std::string& uid) const { return held_.at(uid).row.exact; }
    int32_t GroupID(const std::string& uid) const { return held_.at(uid).row.group; }
    // the id of a scheduler name, -1 for a name no driver has carried (a sweep of it selects nothing)
    int32_t SchedulerID(const std::string& name) const { auto it = schedulers_.find(name); return it == schedulers_.end() ? -1 : it->second; }
    // the interned required affinities by id (an id no driver holds: a program that matches every node), the programs of a
    // marker sweep; a driver's id is -1 when its Program matches every node
    std::vector<affinity::Program> AffinityPrograms() const {
        std::vector<affinity::Program> out((size_t)affNext_);
        for (const auto& kv : affProg_) out[(size_t)kv.first] = kv.second;
        return out;
    }
    int32_t AffinityID(const std::string& uid) const { return held_.at(uid).row.affinity; }
    const std::string& UIDAt(int32_t slot) const { return uidAt_.at(slot); }
    // The marker's stale drivers restated on the host from the held pods: scheduler id `scheduler`, creation + timeout < now
    // (exactly), in (creation, slot) order; outside = exact false, a negative quantity or count
    struct StaleRow { std::string UID; int32_t Affinity; bool Outside; ParsedSparkResources Parsed; };
    std::vector<StaleRow> Stale(int32_t scheduler, int64_t timeoutNs, int64_t nowUnixNano) const {
        std::vector<std::pair<std::pair<int64_t, int32_t>, const Held*>> keep;
        for (const auto& kv : held_) {
            const Row& r = kv.second.row;
            if (r.scheduler == scheduler && (__int128)r.creation + (__int128)timeoutNs < (__int128)nowUnixNano)
                keep.push_back({{r.creation, kv.second.slot}, &kv.second});
        }
        std::sort(keep.begin(), keep.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
        std::vector<StaleRow> out;
        for (const auto& k : keep) {
            const Row& r = k.second->row;
            bool outside = !r.exact || r.count < 0;
            for (int d = 0; d < 6; ++d) outside = outside || r.q[d] < 0;
            out.push_back(StaleRow{k.second->pod.UID, r.affinity, outside, k.second->parsed});
        }
        return out;
    }

    void Flush(gangpack::Device& dev) {
        Grow(size_.n_slots, next_);
        Grow(size_.n_groups, (int64_t)groups_.size());
        Grow(size_.n_schedulers, (int64_t)schedulers_.size());
        std::vector<int32_t> slot, sched, group, count, aff;
        std::vector<uint8_t> present, exact;
        std::vector<int64_t> creation, q[6];
        auto row = [&](int32_t s) {
            const Row r = record(s);
            slot.push_back(s); present.push_back(r.present); exact.push_back(r.exact); creation.push_back(r.creation);
            sched.push_back(r.scheduler); group.push_back(r.group); count.push_back(r.count); aff.push_back(r.affinity);
            for (int k = 0; k < 6; ++k) q[k].push_back(r.q[k]);
        };
        if (Replaying()) {
            sent_.clear();
            for (const auto& kv : uidAt_) row(kv.first);
        } else {
            for (int32_t s : dirty_) {
                auto it = sent_.find(s);
                if (!(record(s) == (it == sent_.end() ? Row{} : it->second))) row(s);
            }
        }
        gp_driver_delta d{(int32_t)slot.size(), 0, slot.data(), present.data(), creation.data(), sched.data(), group.data(),
                          q[0].data(), q[1].data(), q[2].data(), q[3].data(), q[4].data(), q[5].data(), count.data(), exact.data(),
                          aff.data()};
        Send(dev, gp_driver_table_reset, "gp_driver_table_reset", gp_driver_table_update, "gp_driver_table_update",
             slot.empty() ? nullptr : &d);
        for (int32_t s : slot) sent_[s] = record(s);
        dirty_.clear();
    }

private:
    struct Row {
        bool present = false;
        int64_t creation = 0;
        int32_t scheduler = 0, group = -1;
        int64_t q[6] = {0, 0, 0, 0, 0, 0};
        int32_t count = 0;
        bool exact = false;
        int32_t affinity = -1;
        bool operator==(const Row& o) const {
            for (int k = 0; k < 6; ++k) if (q[k] != o.q[k]) return false;
            return present == o.present && creation == o.creation && scheduler == o.scheduler && group == o.group && count == o.count &&
                   exact == o.exact && affinity == o.affinity;
        }
    };
    // a canonical key of a Program ("" when it matches every node: no nodeSelector and no required affinity)
    static std::string affinityKey(const affinity::Program& p) {
        if (p.NodeSelector.empty() && !p.HasRequired) return "";
        std::string k;
        auto put = [&](const std::string& x) { k += std::to_string(x.size()); k += ':'; k += x; };
        for (const auto& kv : p.NodeSelector) { put(kv.first); put(kv.second); }
        k += p.HasRequired ? "|R" : "|N";
        for (const auto& t : p.Terms) {
            for (const auto* part : {&t.MatchExpressions, &t.MatchFields}) {
                k += '[';
                for (const auto& r : *part) { put(r.Key); put(r.Operator); k += '('; for (const auto& v : r.Values) put(v); k += ')'; }
                k += ']';
            }
        }
        return k;
    }
    // the program's id, interned with a reference count (the lowest free id reused); -1 for one that matches every node
    int32_t acquire(const affinity::Program& p) {
        const std::string key = affinityKey(p);
        if (key.empty()) return -1;
        auto it = affId_.find(key);
        if (it == affId_.end()) {
            int32_t a;
            if (!affFree_.empty()) { a = *affFree_.begin(); affFree_.erase(affFree_.begin()); }
            else a = affNext_++;
            it = affId_.emplace(key, a).first;
            affProg_[a] = p;
            affRefs_[a] = 0;
        }
        ++affRefs_[it->second];
        return it->second;
    }
    void release(int32_t a) {
        if (a < 0 || --affRefs_[a] > 0) return;
        affId_.erase(affinityKey(affProg_.at(a)));
        affProg_.erase(a);
        affRefs_.erase(a);
        affFree_.insert(a);
    }
    struct Held { int32_t slot; Row row; QueuedDriverPod pod; ParsedSparkResources parsed; };
    static int32_t intern(std::map<std::string, int32_t>& t, const std::string& name) {
        auto it = t.find(name);
        if (it != t.end()) return it->second;
        const int32_t id = (int32_t)t.size();
        t.emplace(name, id);
        return id;
    }
    Row record(int32_t s) const { auto it = uidAt_.find(s); return it == uidAt_.end() ? Row{} : held_.at(it->second).row; }

    std::map<std::string, Held> held_;
    std::map<int32_t, std::string> uidAt_;       // slot -> uid, in slot order
    std::set<int32_t> free_;
    int32_t next_ = 0;
    std::map<std::string, int32_t> schedulers_, groups_;
    std::set<int32_t> dirty_;
    std::map<int32_t, Row> sent_;
    std::map<std::string, int32_t> affId_;       // affinityKey -> id
    std::map<int32_t, affinity::Program> affProg_;
    std::map<int32_t, int32_t> affRefs_;
    std::set<int32_t> affFree_;
    int32_t affNext_ = 0;
};

// What selectDriverNode's FIFO step decides for the requesting driver: fits (result = its packing), failure-fit (-1) or
// failure-earlier-driver (-2); undefinedTies > 0: equal creation times whose order the reference leaves undefined.
struct DriverQueueOutcome {
    int32_t status = -1;                  // >= 0: fits; -1 failure-fit; -2 failure-earlier-driver
    binpack::PackingResult result;
    int32_t undefinedTies = 0;
    bool fromTable = false;               // false: the per-call path answered (a refusal, or a packer the table entry does not take)
};

// fitEarlierDrivers (resource.go:224-262) followed by the requesting driver's own FIFO step, from the resident driver table:
// one flush, one gp_pack_fifo_driver_table over the snapshot of `metadata`, which then holds the usage of every fitted driver
// (the requesting one included).  The requesting driver must be held (SetDriver it from ExtenderArgs.Pod first: an informer
// can lag).  A capacity refusal grows the buffers and calls again; any other refusal, of the flush or of the call, replays the
// table and falls back to
// FilterToEarliestAndSort over drivers.Pods() plus FitEarlierDrivers, the per-call FIFO batch, on the same metadata.  The
// zone-aware packers, whose snapshot is laid out per zone, take that per-call path too.
inline DriverQueueOutcome FitEarlierDriversDriverTable(const binpacker::Binpacker& packer, ResidentDrivers& drivers,
                                                      const std::string& uid, int64_t defaultEnforceAfterNs,
                                                      const std::map<std::string, int64_t>& enforceAfterOverrides,
                                                      int64_t nowUnixNano, const std::vector<std::string>& nodeNames,
                                                      const std::vector<std::string>& executorNodeNames,
                                                      resources::NodeGroupSchedulingMetadata& metadata) {
    gangpack::Device& d = gangpack::Device::Get();
    DriverQueueOutcome out;
    const bool tableForm = !packer.IsSingleAz && packer.Name != binpacker::azAwareTightlyPack;
    bool flushed = false;
    if (tableForm && drivers.Holds(uid)) {
        try {
            drivers.Flush(d);
            flushed = true;
        } catch (const gangpack::Error&) {
        }
    }
    if (flushed) {
        const std::vector<int64_t> enforceAfterNs = drivers.GroupAges(defaultEnforceAfterNs, enforceAfterOverrides);
        d.SetSnapshot(metadata, nodeNames, executorNodeNames);
        int32_t cap = (int32_t)drivers.Size().n_slots + 1, n = 0, ties = 0;
        int64_t ecap = 4 * (int64_t)cap, ne = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            std::vector<int32_t> slots((size_t)cap), driver((size_t)cap), exec((size_t)std::max<int64_t>(ecap, 1));
            std::vector<int64_t> off((size_t)cap + 1);
            gp_driver_queue q{};
            q.requesting_slot = drivers.Slot(uid);
            q.queue_cap = cap;
            q.enforce_after_ns = enforceAfterNs.data();
            q.now_unix_nano = nowUnixNano;
            q.queue_slot = slots.data(); q.exec_out_off = off.data(); q.n_queued = &n; q.n_executors = &ne; q.undefined_ties = &ties;
            gp_results r{driver.data(), exec.data(), ecap};
            const int st = gp_pack_fifo_driver_table(d.ctx(), &q, (gp_algo)packer.algo, GP_MODE_FIFO_REFERENCE, &r);
            if (st == GP_ERR_CAPACITY && attempt == 0) { cap = std::max(cap, n); ecap = std::max(ecap, ne); continue; }
            if (st != GP_OK) break;
            std::vector<int64_t> cpu(d.n_nodes()), mem(d.n_nodes()), gpu(d.n_nodes());
            d.check(gp_get_snapshot(d.ctx(), cpu.data(), mem.data(), gpu.data()), "gp_get_snapshot");
            for (size_t i = 0; i < d.n_nodes(); ++i) {
                auto& m = metadata.at(d.name((int32_t)i)).AvailableResources;
                m.CPU = cpu[i]; m.Memory = mem[i]; m.NvidiaGPU = gpu[i];
            }
            const int32_t last = n - 1;
            out.status = driver[(size_t)last];
            out.undefinedTies = ties;
            out.fromTable = true;
            if (out.status >= 0) {
                out.result.HasCapacity = true;
                out.result.DriverNode = d.name(out.status);
                for (int64_t t = off[(size_t)last]; t < off[(size_t)last + 1]; ++t) out.result.ExecutorNodes.push_back(d.name(exec[(size_t)t]));
            }
            return out;
        }
    }
    if (tableForm && drivers.Holds(uid)) {       // refused (the update or the call): resend the whole table, then answer with
        drivers.Replay();                        // the per-call path
        drivers.Flush(d);
    }
    // the per-call path: FilterToEarliestAndSort over the listed drivers, shouldSkipDriverFifo, the FIFO batch
    const std::vector<QueuedDriverPod> pods = drivers.Pods();
    const QueuedDriverPod* me = nullptr;
    for (const auto& p : pods) if (p.UID == uid) me = &p;
    if (!me) throw gangpack::Error(GP_ERR_INVALID, "FitEarlierDriversDriverTable: the requesting driver is not held (SetDriver it first)");
    const std::vector<int64_t> enforceAfterNs = drivers.GroupAges(defaultEnforceAfterNs, enforceAfterOverrides);
    std::vector<PendingDriver> queue;
    const std::vector<QueuedDriverPod> earlier = FilterToEarliestAndSort(*me, pods);
    for (size_t j = 0; j < earlier.size(); ++j) {
        const auto& p = earlier[j];
        if (!drivers.Exact(p.UID)) throw gangpack::Error(GP_ERR_UNREPRESENTABLE, "FitEarlierDriversDriverTable: a queued driver is outside the exact-int64 model (run the Go loop)");
        const int32_t g = drivers.GroupID(p.UID);
        const __int128 created = (__int128)p.CreationSeconds * 1000000000LL;
        queue.push_back(drivers.Pending(p.UID, created > (__int128)nowUnixNano - (__int128)enforceAfterNs.at((size_t)g)));
        if (j > 0 && p.CreationSeconds == earlier[j - 1].CreationSeconds) ++out.undefinedTies;
    }
    if (!drivers.Exact(uid)) throw gangpack::Error(GP_ERR_UNREPRESENTABLE, "FitEarlierDriversDriverTable: the driver is outside the exact-int64 model (run the Go loop)");
    if (!FitEarlierDrivers(packer, queue, nodeNames, executorNodeNames, metadata)) { out.status = -2; return out; }
    std::vector<binpack::PackingResult> res;
    FitEarlierDrivers(packer, {drivers.Pending(uid, false)}, nodeNames, executorNodeNames, metadata, &res);
    out.result = res[0];
    out.status = res[0].HasCapacity ? d.index(res[0].DriverNode) : -1;
    return out;
}

inline std::vector<UnschedulablePodMarker::StaleOutcome> UnschedulablePodMarker::DoesPodsExceedClusterCapacity(
        ResidentDrivers& drivers, const std::string& schedulerName, int64_t timeoutNs, int64_t nowUnixNano,
        const std::vector<std::string>& names, resources::ResidentNodes& nodes, affinity::ResidentLabels& labels,
        ResidentOverheadComputer& overhead, const std::vector<std::string>& zones) const {
    gangpack::Device& dev = gangpack::Device::Get();
    overhead.Flush(dev);
    labels.Flush(dev);
    nodes.Flush(dev);
    drivers.Flush(dev);
    const std::vector<affinity::Program> programs = drivers.AffinityPrograms();
    const int32_t scheduler = drivers.SchedulerID(schedulerName);
    std::vector<StaleOutcome> out;
    fellBack_ = false;
    {
        const resources::NodeTableLabels z(labels, zones, "", {});
        MarkerNodeTable t(names, nodes, overhead, z);
        const affinity::Encoded e = labels.EncodePrograms(names, programs);
        const gp_node_affinities p = e.Programs();
        for (;;) {
            const int32_t cap = staleCap_;
            std::vector<int32_t> slot((size_t)cap + 1);
            std::vector<uint8_t> exceeds((size_t)cap + 1), outcome((size_t)cap + 1);
            int32_t n = 0;
            const gp_stale_sweep sw{scheduler, cap, timeoutNs, nowUnixNano, slot.data(), exceeds.data(), outcome.data(), &n};
            const gp_status st = gp_exceeds_cluster_capacity_driver_table(dev.ctx(), &t.nd, &p, &sw, Packer());
            if (st == GP_ERR_CAPACITY && n > cap) { staleCap_ = n; continue; }
            if (st != GP_OK) break;
            for (int32_t i = 0; i < n; ++i) out.push_back(StaleOutcome{drivers.UIDAt(slot[(size_t)i]), exceeds[(size_t)i] != 0, outcome[(size_t)i]});
            return out;
        }
    }
    // refused: replay the four tables and answer per call over the held pods
    fellBack_ = true;
    overhead.Replay();
    labels.Replay();
    nodes.Replay();
    drivers.Replay();
    drivers.Flush(dev);
    const std::vector<ResidentDrivers::StaleRow> stale = drivers.Stale(scheduler, timeoutNs, nowUnixNano);
    std::vector<affinity::Program> progs = programs;
    progs.push_back(affinity::Program{});              // matches every node: the drivers with affinity -1
    std::vector<AffinityStaleDriver> answered;
    for (const auto& r : stale) {
        if (r.Outside) continue;
        AffinityStaleDriver d;
        const ParsedSparkResources& x = r.Parsed;
        d.DriverResources = resources::CreateResources(x.DriverCPUMilli, x.DriverMemoryBytes, x.DriverNvidiaGPUs);
        d.ExecutorResources = resources::CreateResources(x.ExecutorCPUMilli, x.ExecutorMemoryBytes, x.ExecutorNvidiaGPUs);
        d.MinExecutorCount = (int)x.MinExecutorCount;
        d.Affinity = r.Affinity < 0 ? (int)programs.size() : r.Affinity;
        answered.push_back(d);
    }
    std::vector<bool> err;
    const std::vector<bool> exceeds = DoesPodsExceedClusterCapacity(names, nodes, labels, overhead, zones, progs, answered, &err);
    size_t j = 0;
    for (const auto& r : stale) {
        if (r.Outside) { out.push_back(StaleOutcome{r.UID, false, 2}); continue; }
        out.push_back(StaleOutcome{r.UID, exceeds[j], err[j] ? 1 : 0});
        ++j;
    }
    return out;
}

}  // namespace extender

// ------------------------------------------------------------------------------------------------
namespace metrics {

// One node of availableNodes (EXT/resource.go:292-295) as ReportCrossZoneMetric reads it: its name and labels.
struct Node {
    std::string Name;
    std::map<std::string, std::string> Labels;
};

// What the three placement reporters selectDriverNode calls after a successful pack (EXT/resource.go:354-356) would emit:
// ReportInitialDriverExecutorCollocationMetric (internal/metrics/metrics.go:223-252), ReportInitialNodeCountMetrics
// (:254-275, nothing when ExecutorNodes is empty) and ReportCrossZoneMetric (:277-318).  Reported is false for an
// EmptyPackingResult, for which selectDriverNode returns before the metrics.
struct PlacementMetricsResult {
    bool Reported = false;
    std::string CollocationType;           // "no-collocation", "driver-collocated-with-all-executors" or "-some-executors"
    bool NodeCountReported = false;        // ReportInitialNodeCountMetrics returns early when there are no executors
    int64_t ExecutorsPerNode = 0;          // initialExecutorsPerNode
    int64_t NodeCount = 0;                 // initialNodeCount
    int64_t CrossZonePairs = 0;            // crossAzTraffic
    int64_t TotalPairs = 0;                // totalTraffic
    int64_t NumberOfZones = 0;             // applicationZonesCount
};

// The three reporters' inputs for one PackingResult, computed by one gp_placement_metrics call.  availableNodes is the
// Predicate's node list; a driver or executor node that is not in it counts in the pod total and in no zone, as in the
// reference.  The metric zone is the failure-domain.beta.kubernetes.io/zone label, a missing one interned as
// "unknown-zone" (metrics.go:290-294), so it merges with a node literally labelled unknown-zone.  Emitting the counters,
// histograms and gauges stays with the caller.
inline PlacementMetricsResult PlacementMetrics(const binpack::PackingResult& packingResult, const std::vector<Node>& availableNodes) {
    PlacementMetricsResult out;
    if (!packingResult.HasCapacity) return out;
    // node table: availableNodes (instance group 0) then the placed names outside it (instance group -1, zone 0)
    std::unordered_map<std::string, int32_t> index;
    std::unordered_map<std::string, int32_t> zones;
    std::vector<int32_t> zone, group;
    for (const Node& n : availableNodes) {
        if (!index.emplace(n.Name, (int32_t)zone.size()).second) continue;       // a lister's names are unique
        auto it = n.Labels.find(extender::LabelZoneFailureDomain);
        const std::string z = it == n.Labels.end() ? "unknown-zone" : it->second;
        zone.push_back(zones.emplace(z, (int32_t)zones.size()).first->second);
        group.push_back(0);
    }
    auto idx = [&](const std::string& name) {
        auto it = index.find(name);
        if (it != index.end()) return it->second;
        const int32_t i = (int32_t)zone.size();
        index.emplace(name, i);
        zone.push_back(0);
        group.push_back(-1);
        return i;
    };
    int32_t driver = idx(packingResult.DriverNode);
    std::vector<int32_t> execs;
    for (const auto& n : packingResult.ExecutorNodes) execs.push_back(idx(n));
    const int32_t count = (int32_t)execs.size();
    if (execs.empty()) execs.push_back(0);
    const int64_t off[2] = {0, count};
    gp_apps a{};
    a.n_apps = 1;
    a.exe_count = &count;
    a.exec_out_off = off;
    gp_results r{&driver, execs.data(), (int64_t)execs.size()};
    const int32_t n_zones = std::max<int32_t>((int32_t)zones.size(), 1);
    gp_placement_record rec{};
    gangpack::Device& d = gangpack::Device::Get();
    d.check(gp_placement_metrics(d.ctx(), &a, &r, (int32_t)zone.size(), zone.data(), n_zones, group.data(), 1, &rec),
            "gp_placement_metrics");
    static const char* const kTags[3] = {"no-collocation", "driver-collocated-with-all-executors", "driver-collocated-with-some-executors"};
    out.Reported = true;
    out.CollocationType = kTags[rec.collocation];
    out.NodeCountReported = rec.execs_per_node >= 0;
    out.ExecutorsPerNode = out.NodeCountReported ? rec.execs_per_node : 0;
    out.NodeCount = out.NodeCountReported ? rec.distinct_exec_nodes : 0;
    out.CrossZonePairs = rec.cross_zone_pairs;
    out.TotalPairs = rec.total_pairs;
    out.NumberOfZones = rec.n_zones;
    return out;
}

}  // namespace metrics
