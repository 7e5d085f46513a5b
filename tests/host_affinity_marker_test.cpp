// extender::UnschedulablePodMarker::DoesPodsExceedClusterCapacity over affinity programs (one
// gp_exceeds_cluster_capacity_affinity call, overlapping node sets) and affinity::MatchRequiredNodeAffinity
// (gp_match_node_affinity) in the C++ host layer.  The match is checked on hand-derived reference quirks; the sweep against
// the one-class-per-node overload called once per affinity with that affinity's matched nodes as its class, for all five
// `binpack:` values, on clusters where most nodes match several affinities.  Needs an H100.
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

using affinity::Program;
using affinity::Requirement;
using affinity::Term;
using resources::CreateResources;
static const int64_t Gi = 1ll << 30;

static Program Required(std::vector<Term> terms, std::map<std::string, std::string> sel = {}) {
    Program p;
    p.NodeSelector = std::move(sel);
    p.HasRequired = true;
    p.Terms = std::move(terms);
    return p;
}
static Term Exprs(std::vector<Requirement> e, std::vector<Requirement> f = {}) { return Term{std::move(e), std::move(f)}; }

static void Parsing() {
    int64_t v = 0;
    EXPECT(affinity::ParseInt("+5", &v) && v == 5, "+5");
    EXPECT(affinity::ParseInt("007", &v) && v == 7, "007");
    EXPECT(affinity::ParseInt("-0", &v) && v == 0, "-0");
    EXPECT(!affinity::ParseInt(" 5", &v), "' 5'");
    EXPECT(!affinity::ParseInt("9223372036854775808", &v), "2^63");
    EXPECT(affinity::ParseInt("-9223372036854775808", &v) && v == INT64_MIN, "-2^63");
    EXPECT(!affinity::ParseInt("", &v) && !affinity::ParseInt("-", &v) && !affinity::ParseInt("1_0", &v), "syntax");
    EXPECT(affinity::ValidLabelKey("example.com/pool") && affinity::ValidLabelKey("a"), "keys");
    EXPECT(!affinity::ValidLabelKey("/a") && !affinity::ValidLabelKey("a/b/c") && !affinity::ValidLabelKey("-a") &&
           !affinity::ValidLabelKey("Example.com/a") && !affinity::ValidLabelKey(std::string(64, 'a')), "bad keys");
    EXPECT(affinity::ValidLabelValue("") && !affinity::ValidLabelValue("-1") && !affinity::ValidLabelValue("+7"), "values");
}

static void Quirks() {
    const std::vector<affinity::Node> nodes = {{"n0", {{"zone", "a"}, {"gpus", "8"}}}, {"n1", {{"zone", "b"}, {"gpus", "x"}}}, {"n2", {}}};
    std::vector<Program> ps = {
        Required({}),                                                                // empty required affinity: no node
        Required({Exprs({{"gpus", "NotIn", {"8"}}})}),                               // NotIn on an absent key matches
        Required({Exprs({{"zone", "Bogus", {}}})}, {{"zone", "a"}}),                 // the selector masks the parse error
        Required({Exprs({{"zone", "In", {}}}), Exprs({{"zone", "In", {"a"}}})}),     // an error only where no term matched
        Required({Exprs({{"gpus", "Gt", {"4"}}})}),                                  // a value that does not parse: no match
        Required({Exprs({{"gpus", "Gt", {"-1"}}})}),                                 // a negative bound is no label value
        Required({Exprs({}, {{"metadata.name", "In", {"n1"}}})}),
        Required({Exprs({}, {{"spec.other", "In", {""}}})}),                         // any other field reads ""
        Program{}};                                                                  // no required affinity: every node
    const std::vector<std::vector<int32_t>> want = {{}, {1, 2}, {}, {0}, {0}, {}, {1}, {0, 1, 2}, {0, 1, 2}};
    const std::vector<bool> wantFailed = {false, false, true, true, false, true, false, false, false};
    const affinity::MatchResult r = affinity::MatchRequiredNodeAffinity(nodes, ps);
    for (size_t a = 0; a < ps.size(); ++a) {
        char label[48]; std::snprintf(label, sizeof label, "quirk program %zu", a);
        EXPECT(r.Matched[a] == want[a] && r.Failed[a] == wantFailed[a], label);
    }
}

static void Sweep(std::mt19937_64& rng, const char* name, int n, int nZones) {
    auto U = [&](int64_t lo, int64_t hi) { return (int64_t)(lo + (int64_t)(rng() % (uint64_t)(hi - lo + 1))); };
    resources::NodeGroupSchedulingMetadata md;
    std::vector<affinity::Node> nodes;
    for (int i = 0; i < n; ++i) {
        affinity::Node nd;
        nd.Name = "n" + std::to_string(i);
        nd.Labels = {{"ig", "g" + std::to_string(U(0, 3))}, {"zone", "z" + std::to_string(U(0, nZones - 1))},
                     {"type", U(0, 2) == 0 ? "gpu" : "cpu"}};
        resources::NodeSchedulingMetadata m;
        int64_t sc = U(1, 32) * 1000, sm = U(1, 64) * Gi, sg = U(0, 3) == 0 ? U(1, 4) : 0;
        if (U(0, 19) == 0) sc = -U(1, 2000);
        m.SchedulableResources = m.AvailableResources = CreateResources(sc, sm, sg);
        m.ZoneLabel = nd.Labels["zone"];
        md[nd.Name] = m;
        nodes.push_back(nd);
    }
    std::vector<Program> ps = {Program{}};
    for (int k = 0; k < 4; ++k) { Program p; p.NodeSelector = {{"ig", "g" + std::to_string(k)}}; ps.push_back(p); }
    ps.push_back(Required({Exprs({{"ig", "In", {"g0", "g1", "g2"}}})}));
    ps.push_back(Required({Exprs({{"type", "NotIn", {"gpu"}}})}));
    ps.push_back(Required({Exprs({{"ig", "In", {"g3"}}}), Exprs({{"type", "In", {"gpu"}}})}));
    ps.push_back(Required({Exprs({{"ig", "In", {"g1"}}, {"zone", "In", {"z0"}}})}));
    ps.push_back(Required({Exprs({{"zone", "In", {"bad value"}}})}, {{"ig", "g2"}}));      // an error on the g2 nodes
    const affinity::MatchResult match = affinity::MatchRequiredNodeAffinity(nodes, ps);
    const binpacker::Binpacker& packer = *binpacker::SelectBinpacker(name);
    const extender::UnschedulablePodMarker marker(packer);
    std::vector<extender::UnschedulablePodMarker::AffinityStaleDriver> drivers;
    for (int q = 0; q < 80; ++q) {
        extender::UnschedulablePodMarker::AffinityStaleDriver d;
        d.DriverResources = CreateResources(U(0, 4) * 500, U(0, 4) * Gi, U(0, 5) == 0 ? 1 : 0);
        d.ExecutorResources = CreateResources(U(0, 4) * 1000, U(0, 8) * (Gi / 2), U(0, 5) == 0 ? 1 : 0);
        d.Affinity = (int)U(0, (int64_t)ps.size() - 1);
        d.MinExecutorCount = (int)U(0, 2 * n);
        drivers.push_back(d);
    }
    std::vector<bool> affErr;
    const std::vector<bool> got = marker.DoesPodsExceedClusterCapacity(md, nodes, ps, drivers, &affErr);
    char label[96];
    for (size_t i = 0; i < drivers.size(); ++i) {
        const auto& d = drivers[i];
        std::snprintf(label, sizeof label, "%s n=%d driver %zu", name, n, i);
        EXPECT(affErr[i] == match.Failed[(size_t)d.Affinity], label);
        if (affErr[i]) continue;
        std::unordered_map<std::string, int32_t> nodeClass;
        for (int32_t j : match.Matched[(size_t)d.Affinity]) nodeClass[nodes[(size_t)j].Name] = 0;
        extender::UnschedulablePodMarker::StaleDriver one{d.DriverResources, d.ExecutorResources, d.MinExecutorCount, 0};
        const std::vector<bool> want = marker.DoesPodsExceedClusterCapacity(md, nodeClass, 1, {one});
        EXPECT(got[i] == want[0], label);
    }
}

int main() {
    Parsing();
    Quirks();
    std::mt19937_64 rng(4411);
    for (const char* name : {binpacker::tightlyPack, binpacker::distributeEvenly, binpacker::azAwareTightlyPack,
                             binpacker::SingleAzTightlyPack, binpacker::SingleAzMinimalFragmentation})
        for (int n : {6, 120, 2000}) Sweep(rng, name, n, 3);
    if (failures) { std::printf("%d FAILED\n", failures); return 1; }
    std::printf("host_affinity_marker_test: all passed\n");
    return 0;
}
