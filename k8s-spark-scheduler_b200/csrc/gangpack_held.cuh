// gangpack_held.cuh -- private to libgangpack: what the snapshot of a gp_ctx holds, changed only by the transitions below, and
// the requirements the C ABI entries check against it (DESIGN.md §5).  Free of CUDA: tests/held_state_test.cpp runs it on the host.
#pragma once

#include "gangpack.h"

#include <vector>

struct Need { gp_status status; const char* what; };   // a requirement's answer: GP_OK, or the refusal and the text after `who: `

class Held {
public:
    enum class Layout { None, Snapshot, SnapshotDevice, Cluster, Zones, ZonesGroups };   // the call that laid it out
    enum class Sched { None, Efficiency, Full };    // SchedulableResources: none, for gp_packing_efficiency alone, for all

    // ---- transitions
    // gp_set_snapshot, before its validation overwrites the host copy (v_owner / v_pos); a refusal leaves the rest
    void host_copy_overwritten() { host_copy_ = false; }
    // Every layout entry past its last refusal, before its first write to a snapshot buffer or zoneprep: until the new
    // layout is installed nothing is held, so one that fails with a CUDA error leaves no snapshot over freed buffers
    void commit() { *this = Held(); }
    // installed once the layout is enqueued without error
    void laid_out_snapshot() { layout_ = Layout::Snapshot; host_copy_ = true; }
    // tail: the stream of the layout when a gp_pack_batch_device there may start before it ends (GP_CFG_ASYNC_SNAPSHOT)
    void laid_out_device(const void* tail) { layout_ = Layout::SnapshotDevice; tail_ = tail; }
    void laid_out_cluster() { layout_ = Layout::Cluster; sched_ = Sched::Efficiency; }
    // orders: the undivided orders (device pointers) and n_zones.  n_ig > 0: gp_prepare_cluster_zones_groups, whose words
    // [4 * (n_ig + 1)] are group_off, n_zones (n_ig used), undivided exec_off and drv_off of every instance group
    void laid_out_zones(int32_t kind, const gp_az_orders& orders, int32_t n_ig, const int32_t* words) {
        layout_ = n_ig > 0 ? Layout::ZonesGroups : Layout::Zones; sched_ = Sched::Full; kind_ = kind; orders_ = orders; n_ig_ = n_ig;
        words_.assign(words, words + (n_ig > 0 ? 4 * ((size_t)n_ig + 1) : 0));
    }
    void schedulable_set() { sched_ = Sched::Full; }
    // every entry that enqueues device work takes the tail: the layout is the last work on its stream only until then
    const void* take_tail() { const void* t = tail_; tail_ = nullptr; return t; }

    // ---- requirements
    Need snapshot(const char* what = "gp_set_snapshot first") const { return layout_ == Layout::None ? Need{GP_ERR_NO_SNAPSHOT, what} : ok(); }
    Need full_sched() const { return sched_ == Sched::Full ? ok() : invalid("gp_set_schedulable first (the efficiencies need SchedulableResources)"); }
    Need efficiency_sched() const { return sched_ != Sched::None ? ok() : invalid("no SchedulableResources (gp_set_schedulable, gp_prepare_cluster or gp_prepare_cluster_zones first)"); }
    // the single-instance-group zone entries read the whole snapshot as one instance group's zones
    Need one_instance_group() const {
        return layout_ == Layout::ZonesGroups && n_ig_ > 1 ? invalid("the snapshot holds several instance groups (gp_prepare_cluster_zones_groups): "
                                                                     "drain them with gp_pack_fifo_zones_groups(groups == NULL)") : ok();
    }
    // the az-aware entries' orders == NULL: orders()
    Need az_orders() const {
        if (one_instance_group().status != GP_OK) return one_instance_group();
        if (layout_ != Layout::Zones && layout_ != Layout::ZonesGroups) return invalid("NULL apps/orders/results");
        return kind_ == GP_LAYOUT_AZ_AWARE ? ok() : invalid("orders == NULL needs a gp_prepare_cluster_zones(GP_LAYOUT_AZ_AWARE) snapshot; "
                                                            "this one is GP_LAYOUT_SINGLE_AZ (no trailing group, no undivided orders)");
    }
    // gp_pack_fifo_zones_groups(groups == NULL): groups()
    Need groups_layout(bool az_aware) const {
        if (layout_ != Layout::ZonesGroups) return invalid("groups == NULL needs the layout of gp_prepare_cluster_zones_groups; the snapshot was laid out by another call since");
        if (az_aware == (kind_ == GP_LAYOUT_AZ_AWARE)) return ok();
        return invalid(az_aware ? "az-aware-tightly-pack needs a GP_LAYOUT_AZ_AWARE layout; the held one is GP_LAYOUT_SINGLE_AZ"
                                : "the single-AZ packers need a GP_LAYOUT_SINGLE_AZ layout; the held one is GP_LAYOUT_AZ_AWARE");
    }
    // the host copy to check caller-given undivided orders (groups: instance groups) against
    Need host_copy(bool groups) const {
        if (host_copy_) return ok();
        return invalid(groups ? "the snapshot must be laid out by gp_set_snapshot (after gp_set_snapshot_device / gp_prepare_cluster* there is "
                                "no host copy of the layout to check the instance groups against)"
                              : "the snapshot must be laid out by gp_set_snapshot (after gp_set_snapshot_device / gp_prepare_cluster there is "
                                "no host copy of the layout to check the undivided orders against)");
    }

    const gp_az_orders* orders() const { return &orders_; }
    // groups_layout(): every instance group's words and the undivided orders, as gp_pack_fifo_zones_groups takes them
    gp_instance_groups groups() const {
        const int32_t* w = words_.data();
        const size_t g1 = (size_t)n_ig_ + 1;
        return {n_ig_, w, w + g1, w + 2 * g1, orders_.exec_order, w + 3 * g1, orders_.drv_order};
    }

private:
    static Need ok() { return {GP_OK, nullptr}; }
    static Need invalid(const char* what) { return {GP_ERR_INVALID, what}; }

    Layout layout_ = Layout::None;
    bool host_copy_ = false;                 // v_owner / v_pos describe the layout
    Sched sched_ = Sched::None;
    int32_t kind_ = -1, n_ig_ = 0;           // Zones: the gp_zone_layout_kind; ZonesGroups: also n_instance_groups
    gp_az_orders orders_{};                  // Zones, ZonesGroups
    std::vector<int32_t> words_;             // ZonesGroups
    const void* tail_ = nullptr;
};
