// binpack::AzAwareTightlyPack (az_aware_pack_tightly.go:27-38) in the C++ host layer, one decision at a time -- one
// upload of the az-aware layout and one gp_pack_batch_az_aware call each -- against orc_binpack with the az-aware packer,
// the string-keyed literal restatement, on the unmodified cluster: driver node and ExecutorNodes of every application.
// The clusters have separate driver / executor orders, zones with one kind of candidate only and applications larger
// than any single zone, so the undivided fallback places some of them; one trial has 70 candidate zones.  Needs an H100.
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

// one trial: n nodes over `zones` zones, q independent decisions; returns how many of them the fallback placed
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
    int fell_back = 0, placed = 0, mismatches = 0;
    for (int i = 0; i < q; ++i) {
        const orc_res drv{U(0, 4) * 500, U(0, 2) * Gi, 0}, exe{U(1, 4) * 500, U(1, 4) * Gi, 0};
        const int32_t cnt = (int32_t)(U(0, 5) == 0 ? U(10, 4 * n / zones + 10) : U(0, 6));      // some larger than a zone holds
        int32_t od = -9;
        std::vector<int32_t> oe((size_t)std::max(cnt, 1), -1);
        const int fits = orc_binpack(cl, ORC_AZ_AWARE_TIGHTLY_PACK, &drv, &exe, cnt, cd.data(), (int32_t)cd.size(), ce.data(),
                                     (int32_t)ce.size(), 1, &od, oe.data(), nullptr);
        const binpack::PackingResult r = binpack::AzAwareTightlyPack(CreateResources(drv.cpu, drv.mem, 0), CreateResources(exe.cpu, exe.mem, 0),
                                                                     cnt, dorder, eorder, md);
        bool same = r.HasCapacity == (fits != 0);
        if (same && fits) {
            same = r.DriverNode == names[(size_t)od] && r.ExecutorNodes.size() == (size_t)cnt;
            for (int t = 0; same && t < cnt; ++t) same = r.ExecutorNodes[(size_t)t] == names[(size_t)oe[(size_t)t]];
        }
        if (!same && mismatches++ < 3) std::printf("az-aware mismatch: %s, application %d\n", label, i);
        EXPECT(same, "binpack::AzAwareTightlyPack == orc_binpack(ORC_AZ_AWARE_TIGHTLY_PACK)");
        gp_stats st{};
        gangpack::Device::Get().check(gp_last_stats(gangpack::Device::Get().ctx(), &st), "gp_last_stats");
        fell_back += (int)st.scan_path_apps;                  // 0 or 1: the fallback ran for this decision
        placed += (r.HasCapacity && st.scan_path_apps == 1) ? 1 : 0;
    }
    // the metadata is the caller's and independent decisions leave it as it was
    std::vector<int64_t> fc((size_t)n), fm((size_t)n), fg((size_t)n);
    orc_cluster_get_available(cl, fc.data(), fm.data(), fg.data());
    for (int i = 0; i < n; ++i) {
        const auto& a = md[names[(size_t)i]].AvailableResources;
        EXPECT(a.CPU == fc[(size_t)i] && a.Memory == fm[(size_t)i] && fc[(size_t)i] == cpu[(size_t)i], "availability unchanged");
    }
    EXPECT(fell_back >= placed, "scan_path_apps counts the fallback's decisions");
    orc_cluster_free(cl);
    return placed;
}

int main() {
    std::mt19937_64 rng(5151);
    int placed = 0;
    for (int trial = 0; trial < 16; ++trial) {
        char label[64]; std::snprintf(label, sizeof label, "trial %d", trial);
        placed += Trial(rng, (int)(12 + rng() % 60), (int)(1 + rng() % 5), 24, label);
    }
    placed += Trial(rng, 3 * 70, 70, 30, "70 zones");
    EXPECT(placed > 0, "the undivided fallback placed applications");
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_az_aware_batch_test: all passed (the fallback placed %d applications)\n", placed);
    return 0;
}
