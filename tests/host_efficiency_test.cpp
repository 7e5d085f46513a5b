// extender::ComputeAvgPackingEfficiencyForResult (one gp_packing_efficiency call) in the C++ host layer against the host
// reference binpack::ComputeAvgPackingEfficiency(md, computePackingEfficiency(..., ReservedOf(...)) over every node), which
// sums in the metadata map's iteration order like the Go code: within the recursive-summation bound
// gamma_{m-1} * sum|t| / len + 2 ulp on random clusters (overcommitted nodes, zero and negative schedulable values, mixed
// GPU and non-GPU nodes, CPU not a multiple of 1000), and bit for bit on clusters where every partial sum is exact
// (power-of-two schedulable values).  Placements are random and need not be feasible.  Needs an H100.
#include <cmath>
#include <cstdio>
#include <random>
#include <string>
#include <vector>

#include "gangpack_host.hpp"

static int failures = 0;
#define EXPECT(cond, msg)                                                            \
    do {                                                                             \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

using resources::CreateResources;
using resources::NodeGroupSchedulingMetadata;
static const int64_t Gi = 1ll << 30;

// the host reference: every node of md, reserved from the placement (driver only for minimal-fragmentation)
static binpack::AvgPackingEfficiency HostReference(const NodeGroupSchedulingMetadata& md, const binpack::PackingResult& r,
                                                   const resources::Resources& drv, const resources::Resources& exe, bool minfrag,
                                                   std::vector<binpack::PackingEfficiency>* effs) {
    resources::NodeGroupResources reserved;
    if (minfrag) reserved[r.DriverNode] = drv;
    else reserved = binpack::ReservedOf(drv, exe, r);
    effs->clear();
    for (const auto& kv : md) effs->push_back(binpack::computePackingEfficiency(kv.first, kv.second, reserved));
    return binpack::ComputeAvgPackingEfficiency(md, *effs);
}

static bool WithinBound(double dev, double host, const std::vector<double>& terms, double len) {
    const double u = std::ldexp(1.0, -53);
    const double m = (double)terms.size();
    const double gam = m > 1 ? (m - 1) * u / (1 - (m - 1) * u) : 0.0;
    double abs_sum = 0;
    for (double t : terms) abs_sum += std::fabs(t);
    const double ulp = std::nextafter(std::fabs(host), INFINITY) - std::fabs(host);
    return std::fabs(dev - host) <= gam * abs_sum * (1 + 4 * m * u) / len + 2 * ulp;
}

static void Trial(std::mt19937_64& rng, int n, bool pow2, const char* label) {
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    NodeGroupSchedulingMetadata md;
    std::vector<std::string> names;
    for (int i = 0; i < n; ++i) {
        char buf[16]; std::snprintf(buf, sizeof buf, "n%05d", i);
        names.push_back(buf);
        resources::NodeSchedulingMetadata m;
        int64_t sc, sm, sg;
        if (pow2) {
            sc = 1000ll << U(2, 6); sm = 1ll << U(30, 38); sg = U(0, 9) < 4 ? 1ll << U(0, 3) : 0;
            m.AvailableResources = CreateResources(sc - 1000 * U(-4, 2 * (sc / 1000)), sm - (1ll << 20) * U(-64, 2 * (sm >> 20)), sg - U(-1, 2 * sg));
        } else {
            sc = U(1, 63) * 1000 + (U(0, 1) ? U(0, 999) : 0);
            if (U(0, 19) == 0) sc = 0; else if (U(0, 19) == 0) sc = -U(1, 2999);
            sm = U(1, 255) * Gi + U(0, 1 << 20);
            if (U(0, 19) == 0) sm = 0; else if (U(0, 19) == 0) sm = -U(1, Gi);
            sg = U(0, 9) < 3 ? U(1, 8) : (U(0, 29) == 0 ? -1 : 0);
            m.AvailableResources = CreateResources(sc - U(-2000, std::max<int64_t>(sc, 0) + 5000), sm - U(-Gi, std::max<int64_t>(sm, 0) + 4 * Gi),
                                                   sg - U(-1, std::max<int64_t>(sg, 0) + 2));
        }
        m.SchedulableResources = CreateResources(sc, sm, sg);
        md[buf] = m;
    }
    for (int q = 0; q < 24; ++q) {
        const bool minfrag = q % 3 == 2;
        binpack::PackingResult r;
        r.HasCapacity = true;
        r.DriverNode = names[(size_t)U(0, n - 1)];
        const int k = (int)U(0, 40);
        for (int t = 0; t < k; ++t) r.ExecutorNodes.push_back(names[(size_t)U(0, n - 1)]);
        const auto drv = CreateResources(U(0, 4) * 1000, U(0, 8) * (1ll << 29), U(0, 1));
        const auto exe = pow2 ? CreateResources(U(0, 3) * 1000, U(0, 16) * (1ll << 28), U(0, 1))
                              : CreateResources(U(1, 8) * 250, U(1, 16) * (1ll << 28) + U(0, 999), U(0, 1));
        const auto dev = extender::ComputeAvgPackingEfficiencyForResult(md, r, drv, exe, minfrag ? GP_MINIMAL_FRAGMENTATION : GP_TIGHTLY_PACK);
        std::vector<binpack::PackingEfficiency> effs;
        const auto host = HostReference(md, r, drv, exe, minfrag, &effs);
        if (pow2) {
            EXPECT(dev.CPU == host.CPU && dev.Memory == host.Memory && dev.GPU == host.GPU && dev.Max == host.Max, label);
            continue;
        }
        std::vector<double> c, m, g, x;
        for (const auto& e : effs) {
            c.push_back(e.CPU); m.push_back(e.Memory); x.push_back(e.Max());
            if (md.at(e.NodeName).SchedulableResources.NvidiaGPU != 0) g.push_back(e.GPU);
        }
        const double len = std::max((double)effs.size(), 1.0);
        EXPECT(WithinBound(dev.CPU, host.CPU, c, len), label);
        EXPECT(WithinBound(dev.Memory, host.Memory, m, len), label);
        EXPECT(g.empty() ? dev.GPU == 1.0 && host.GPU == 1.0 : WithinBound(dev.GPU, host.GPU, g, (double)g.size()), label);
        EXPECT(WithinBound(dev.Max, host.Max, x, len), label);
    }
    // EmptyPackingResult: WorstAvgPackingEfficiency without a device call
    const auto worst = extender::ComputeAvgPackingEfficiencyForResult(md, binpack::EmptyPackingResult(), resources::Zero(), resources::Zero());
    EXPECT(worst.CPU == 0 && worst.Memory == 0 && worst.GPU == 0 && worst.Max == 0, label);
}

int main() {
    std::mt19937_64 rng(7331);
    for (int n : {10, 100, 1000, 10000}) {
        char label[64];
        std::snprintf(label, sizeof label, "random n=%d", n);
        Trial(rng, n, false, label);
        std::snprintf(label, sizeof label, "exact n=%d", n);
        Trial(rng, n, true, label);
    }
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_efficiency_test: all passed\n");
    return 0;
}
