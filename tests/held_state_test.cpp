// CPU-only test of the context's snapshot state (k8s-spark-scheduler_b200/csrc/gangpack_held.cuh): every layout entry,
// completed and failed after its commit point, a refused gp_set_snapshot after each, and gp_set_schedulable, each followed
// by the outcome of every requirement.  The transitions are called in the order the entries call them.  No device.
#include <cstdio>
#include <cstring>
#include <string>

#include "gangpack.h"
#include "gangpack_held.cuh"

static int failures = 0;
#define EXPECT(cond, msg)                                                                   \
    do {                                                                                    \
        if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, msg); ++failures; } \
    } while (0)

static int tail_stream;                    // stands for the stream gp_set_snapshot_device enqueued its layout on
static const int32_t kWords[4 * 4] = {0, 2, 4, 5, 2, 2, 1, 0, 0, 3, 7, 9, 0, 2, 4, 6};   // three instance groups' words

// the entries, as far as the state goes
struct Layout {
    const char* name;
    void (*complete)(Held&);               // every transition of a call whose layout is enqueued without error
};
static const gp_az_orders kOrders{3, 9, nullptr, 6, nullptr};
static const Layout kLayouts[] = {
    {"gp_set_snapshot", [](Held& h) { h.host_copy_overwritten(); h.commit(); h.laid_out_snapshot(); }},
    {"gp_set_snapshot_device", [](Held& h) { h.commit(); h.laid_out_device(&tail_stream); }},
    {"gp_prepare_cluster", [](Held& h) { h.commit(); h.laid_out_cluster(); }},
    {"gp_prepare_cluster_zones(single-AZ)", [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_SINGLE_AZ, kOrders, 0, kWords); }},
    {"gp_prepare_cluster_zones(az-aware)", [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_AZ_AWARE, kOrders, 0, kWords); }},
    {"gp_prepare_cluster_zones_groups(single-AZ, 1)",
     [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_SINGLE_AZ, kOrders, 1, kWords); }},
    {"gp_prepare_cluster_zones_groups(az-aware, 1)",
     [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_AZ_AWARE, kOrders, 1, kWords); }},
    {"gp_prepare_cluster_zones_groups(single-AZ, 3)",
     [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_SINGLE_AZ, kOrders, 3, kWords); }},
    {"gp_prepare_cluster_zones_groups(az-aware, 3)",
     [](Held& h) { h.commit(); h.laid_out_zones(GP_LAYOUT_AZ_AWARE, kOrders, 3, kWords); }},
};
static void refused_set_snapshot(Held& h) { h.host_copy_overwritten(); }   // refused by its validation
static bool set_schedulable(Held& h) {                                      // true: accepted
    if (h.snapshot().status != GP_OK) return false;
    h.schedulable_set();
    return true;
}

// Every requirement's outcome, one character each: '.' met, 'N' GP_ERR_NO_SNAPSHOT, 'I' GP_ERR_INVALID, in the order
// snapshot, full SchedulableResources, efficiency SchedulableResources, one instance group, held az-aware orders, held
// groups layout (single-AZ), held groups layout (az-aware), host copy
static std::string outcomes(const Held& h) {
    const Need n[] = {h.snapshot(), h.full_sched(), h.efficiency_sched(), h.one_instance_group(), h.az_orders(),
                      h.groups_layout(false), h.groups_layout(true), h.host_copy(false)};
    std::string s;
    for (const Need& r : n) s += r.status == GP_OK ? '.' : r.status == GP_ERR_NO_SNAPSHOT ? 'N' : r.status == GP_ERR_INVALID ? 'I' : '?';
    return s;
}
static void expect_outcomes(const Held& h, const char* want, const std::string& step) {
    const std::string got = outcomes(h);
    if (got != want) std::printf("FAIL %s: requirements %s, expected %s\n", step.c_str(), got.c_str(), want);
    failures += got != want;
}

static const char* const kNone = "NII.IIII";
// after each layout of kLayouts: completed, then after a refused gp_set_snapshot, then after gp_set_schedulable
static const char* const kExpect[][3] = {
    {".II.III.", ".II.IIII", "....IIII"},
    {".II.IIII", ".II.IIII", "....IIII"},
    {".I..IIII", ".I..IIII", "....IIII"},
    {"....IIII", "....IIII", "....IIII"},
    {".....III", ".....III", ".....III"},
    {"....I.II", "....I.II", "....I.II"},
    {".....I.I", ".....I.I", ".....I.I"},
    {"...II.II", "...II.II", "...II.II"},
    {"...III.I", "...III.I", "...III.I"},
};

static bool contains(const char* s, const char* part) { return s && std::strstr(s, part); }

int main() {
    static_assert(sizeof(kExpect) / sizeof(kExpect[0]) == sizeof(kLayouts) / sizeof(kLayouts[0]), "one row per layout");
    {
        Held h;
        expect_outcomes(h, kNone, "a new context");
        EXPECT(h.take_tail() == nullptr, "a new context has no layout tail");
        EXPECT(!set_schedulable(h), "gp_set_schedulable needs a snapshot");
        expect_outcomes(h, kNone, "gp_set_schedulable without a snapshot");
    }
    // every layout from every earlier state: the new layout replaces the old one whole, and one that fails after its
    // commit point leaves no snapshot
    const size_t L = sizeof(kLayouts) / sizeof(kLayouts[0]);
    for (size_t before = 0; before <= L; ++before) {
        for (size_t i = 0; i < L; ++i) {
            const std::string from = before < L ? std::string(" after ") + kLayouts[before].name : std::string();
            Held h;
            if (before < L) { kLayouts[before].complete(h); set_schedulable(h); h.take_tail(); }
            kLayouts[i].complete(h);
            const std::string step = std::string(kLayouts[i].name) + from;
            expect_outcomes(h, kExpect[i][0], step);
            refused_set_snapshot(h);
            expect_outcomes(h, kExpect[i][1], step + ", then a refused gp_set_snapshot");
            EXPECT(set_schedulable(h), "gp_set_schedulable is accepted over any snapshot");
            expect_outcomes(h, kExpect[i][2], step + ", then gp_set_schedulable");

            Held f;
            if (before < L) { kLayouts[before].complete(f); set_schedulable(f); }
            f.commit();                                  // every layout commits before its first write; this one fails
            expect_outcomes(f, kNone, std::string(kLayouts[i].name) + " failing after its commit point" + from);
            EXPECT(f.take_tail() == nullptr, "a failed layout leaves no layout tail");
            refused_set_snapshot(f);
            expect_outcomes(f, kNone, "a refused gp_set_snapshot after a failed layout");
        }
    }
    // the layout tail: only gp_set_snapshot_device leaves one, and the next entry takes it
    {
        Held h;
        kLayouts[1].complete(h);
        EXPECT(h.take_tail() == &tail_stream, "gp_set_snapshot_device leaves its stream as the layout tail");
        EXPECT(h.take_tail() == nullptr, "the entry after it takes the tail");
        h.commit(); h.laid_out_device(nullptr);
        EXPECT(h.take_tail() == nullptr, "without GP_CFG_ASYNC_SNAPSHOT there is no tail");
        kLayouts[1].complete(h);
        kLayouts[0].complete(h);
        EXPECT(h.take_tail() == nullptr, "a later layout clears the tail");
    }
    // what the held layouts give: the orders, the instance groups and their words, and the refusals' texts
    {
        Held h;
        kLayouts[8].complete(h);
        EXPECT(h.orders()->n_zones == 3 && h.orders()->n_exec == 9 && h.orders()->n_drv == 6, "held az-aware orders");
        const gp_instance_groups g = h.groups();
        EXPECT(g.n_instance_groups == 3 && std::memcmp(g.group_off, kWords, sizeof(kWords)) == 0 &&
                   g.n_zones == g.group_off + 4 && g.exec_off == g.group_off + 8 && g.drv_off == g.group_off + 12, "held instance-group words");
        EXPECT(contains(h.az_orders().what, "several instance groups"), "orders == NULL over several instance groups");
        EXPECT(contains(h.groups_layout(false).what, "the held one is GP_LAYOUT_AZ_AWARE"), "single-AZ packer, az-aware layout");
        kLayouts[7].complete(h);
        EXPECT(contains(h.groups_layout(true).what, "the held one is GP_LAYOUT_SINGLE_AZ"), "az-aware packer, single-AZ layout");
        kLayouts[3].complete(h);
        EXPECT(contains(h.az_orders().what, "this one is GP_LAYOUT_SINGLE_AZ"), "orders == NULL over a single-AZ zone layout");
        EXPECT(contains(h.groups_layout(false).what, "laid out by another call since"), "groups == NULL after another layout");
        kLayouts[2].complete(h);
        EXPECT(contains(h.az_orders().what, "NULL apps/orders/results"), "orders == NULL without a zone layout");
        EXPECT(contains(h.full_sched().what, "gp_set_schedulable first"), "full SchedulableResources");
        EXPECT(contains(h.host_copy(false).what, "laid out by gp_set_snapshot") &&
                   contains(h.host_copy(false).what, "undivided orders"), "host copy for the order checks");
        EXPECT(contains(h.host_copy(true).what, "laid out by gp_set_snapshot") &&
                   contains(h.host_copy(true).what, "instance groups"), "host copy for the instance-group checks");
        h.commit();
        EXPECT(contains(h.snapshot().what, "gp_set_snapshot first") && contains(h.snapshot("no snapshot").what, "no snapshot"),
               "the snapshot requirement's text");
        EXPECT(contains(h.efficiency_sched().what, "no SchedulableResources"), "efficiency SchedulableResources");
    }
    if (failures) { std::printf("%d failures\n", failures); return 1; }
    std::printf("all passed\n");
    return 0;
}
