// extender::FitEarlierDrivers with "az-aware-tightly-pack" (one gp_pack_fifo_az_aware call for the whole queue; above 64
// candidate zones the per-driver loop) against orc_fifo, the string-keyed literal loop over AzAwareTightlyPack
// (az_aware_pack_tightly.go:27-38): placements, blocking and the metadata left behind.  The queues are built so that the
// undivided fallback places drivers: separate driver / executor orders, zones with one kind of candidate only, and
// applications larger than any single zone.  Needs an H100.
#include <algorithm>
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "gangpack_host.hpp"
#include "gangpack_oracle.h"   // the CPU oracle is the checker here (tests/ may link it; the product never does)

static int failures = 0;
#define EXPECT(cond, msg)                                                            \
    do {                                                                             \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

using resources::CreateResources;
using resources::NodeGroupSchedulingMetadata;
using resources::NodeSchedulingMetadata;
typedef std::vector<std::string> Names;
static const int64_t Gi = 1ll << 30;

// one trial: n nodes over `zones` zones; returns gp_stats.scan_path_apps of the last device call (with at most 64 candidate
// zones: the applications for which the undivided fallback ran)
static int Trial(std::mt19937_64& rng, int n, int zones, int q, const char* label) {
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    std::vector<std::string> names, zone;
    std::vector<int64_t> cpu, mem, gpu, scpu, smem, sgpu;
    for (int i = 0; i < n; ++i) {
        char buf[16]; std::snprintf(buf, sizeof buf, "n%04d", i);
        const int64_t sc = U(4, 16) * 1000, sm = U(8, 32) * Gi;
        names.push_back(buf);
        zone.push_back("z" + std::to_string(i < zones ? i : U(0, zones - 1)));    // every zone has a node
        cpu.push_back(U(0, sc / 500) * 500); mem.push_back(U(0, sm / Gi) * Gi); gpu.push_back(0);
        scpu.push_back(sc); smem.push_back(sm); sgpu.push_back(0);
    }
    // zone z0: driver candidates only; zone z1: executor candidates only (when there are more than two zones)
    Names dorder, eorder;
    {
        Names perm = names;
        std::shuffle(perm.begin(), perm.end(), rng);
        for (size_t i = 0; i < perm.size(); ++i) {
            const std::string& z = zone[(size_t)std::stoi(perm[i].substr(1))];
            if (!(zones > 2 && z == "z1") && U(0, 9) < 8) dorder.push_back(perm[i]);
        }
        std::shuffle(perm.begin(), perm.end(), rng);
        for (size_t i = 0; i < perm.size(); ++i) {
            const std::string& z = zone[(size_t)std::stoi(perm[i].substr(1))];
            if (!(zones > 2 && z == "z0") && U(0, 9) < 9) eorder.push_back(perm[i]);
        }
    }
    std::vector<const char*> cn, cz, cd, ce;
    for (auto& s : names) cn.push_back(s.c_str());
    for (auto& s : zone) cz.push_back(s.c_str());
    for (auto& s : dorder) cd.push_back(s.c_str());
    for (auto& s : eorder) ce.push_back(s.c_str());
    std::vector<orc_res> drv((size_t)q), exe((size_t)q);
    std::vector<int32_t> cnt((size_t)q);
    std::vector<uint8_t> young((size_t)q);
    std::vector<int64_t> off((size_t)q + 1, 0);
    std::vector<extender::PendingDriver> queue((size_t)q);
    for (int i = 0; i < q; ++i) {
        drv[(size_t)i] = {U(0, 4) * 500, U(0, 2) * Gi, 0}; exe[(size_t)i] = {U(1, 4) * 500, U(1, 4) * Gi, 0};
        cnt[(size_t)i] = (int32_t)(U(0, 7) == 0 ? U(10, 4 * n / zones + 10) : U(0, 6));      // some larger than a zone holds
        young[(size_t)i] = (uint8_t)(U(0, 9) != 0);
        off[(size_t)i + 1] = off[(size_t)i] + cnt[(size_t)i];
        auto& a = queue[(size_t)i];
        a.Resources.DriverResources = CreateResources(drv[(size_t)i].cpu, drv[(size_t)i].mem, 0);
        a.Resources.ExecutorResources = CreateResources(exe[(size_t)i].cpu, exe[(size_t)i].mem, 0);
        a.Resources.MinExecutorCount = cnt[(size_t)i]; a.SkipIfNoFit = young[(size_t)i] != 0;
    }
    NodeGroupSchedulingMetadata md;
    for (int i = 0; i < n; ++i) {
        NodeSchedulingMetadata m;
        m.AvailableResources = CreateResources(cpu[(size_t)i], mem[(size_t)i], 0);
        m.SchedulableResources = CreateResources(scpu[(size_t)i], smem[(size_t)i], 0);
        m.ZoneLabel = zone[(size_t)i];
        md[names[(size_t)i]] = m;
    }
    orc_cluster* cl = orc_cluster_new(n, cn.data(), cpu.data(), mem.data(), gpu.data(), scpu.data(), smem.data(), sgpu.data(),
                                      cz.data(), nullptr, nullptr);
    std::vector<int32_t> od((size_t)q, -9), oe((size_t)std::max<int64_t>(off[(size_t)q], 1), -1);
    const int32_t blocked = orc_fifo(cl, ORC_AZ_AWARE_TIGHTLY_PACK, ORC_FIFO_REFERENCE, q, drv.data(), exe.data(), cnt.data(),
                                     young.data(), cd.data(), (int32_t)cd.size(), ce.data(), (int32_t)ce.size(), 0, off.data(),
                                     od.data(), oe.data());
    std::vector<binpack::PackingResult> res;
    const bool ok = extender::FitEarlierDrivers(*binpacker::SelectBinpacker("az-aware-tightly-pack"), queue, dorder, eorder, md, &res);
    bool same = ok == (blocked < 0);
    for (int i = 0; same && i < q; ++i) {
        if (od[(size_t)i] < 0) { same = !res[(size_t)i].HasCapacity; continue; }
        same = res[(size_t)i].HasCapacity && res[(size_t)i].DriverNode == names[(size_t)od[(size_t)i]];
        for (int t = 0; same && t < cnt[(size_t)i]; ++t)
            same = res[(size_t)i].ExecutorNodes[(size_t)t] == names[(size_t)oe[(size_t)(off[(size_t)i] + t)]];
    }
    std::vector<int64_t> fc((size_t)n), fm((size_t)n), fg((size_t)n);
    orc_cluster_get_available(cl, fc.data(), fm.data(), fg.data());
    for (int i = 0; same && i < n; ++i) {
        const auto& a = md[names[(size_t)i]].AvailableResources;
        same = a.CPU == fc[(size_t)i] && a.Memory == fm[(size_t)i] && a.NvidiaGPU == fg[(size_t)i];
    }
    if (!same) std::printf("az-aware fifo mismatch: %s\n", label);
    EXPECT(same, "FitEarlierDrivers(az-aware-tightly-pack) == orc_fifo");
    // applications for which the undivided fallback ran in the one device call (gp_stats.scan_path_apps)
    gp_stats st{};
    gangpack::Device::Get().check(gp_last_stats(gangpack::Device::Get().ctx(), &st), "gp_last_stats");
    orc_cluster_free(cl);
    return (int)st.scan_path_apps;
}

int main() {
    std::mt19937_64 rng(4242);
    int fallbacks = 0;
    for (int trial = 0; trial < 16; ++trial) {
        char label[64]; std::snprintf(label, sizeof label, "trial %d", trial);
        fallbacks += Trial(rng, (int)(12 + rng() % 60), (int)(1 + rng() % 5), 24, label);
    }
    EXPECT(fallbacks > 0, "the undivided fallback ran inside the one-call FIFO loop");
    Trial(rng, 3 * 70, 70, 30, "70 zones");                  // more than 64 candidate zones: the per-driver loop
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_az_aware_test: all passed (fallback ran for %d applications)\n", fallbacks);
    return 0;
}
