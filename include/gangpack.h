/*
 * gangpack.h -- C ABI of libgangpack.so, the H100-native gang-scheduling bin-packer.
 *
 * This is the drop-in boundary for ONE hot path of palantir/k8s-spark-scheduler: what a cgo shim
 * registered in internal/binpacker.binpackFunctions (internal/binpacker/binpack.go:43-49) binds in
 * place of binpack.TightlyPack / binpack.DistributeEvenly
 * (vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg/binpack/pack_tightly.go:25-32,
 *  distribute_evenly.go:25-32; contract binpack.SparkBinPackFunction, binpack.go:43-48) and what a
 * batched fitEarlierDrivers (internal/extender/resource.go:224-262) calls once per Predicate.
 * The reference-side binding is shown in INTEGRATION.md.
 *
 * Conventions
 *  - plain C, plain pointers and sizes; no exceptions cross the boundary; every call returns a
 *    gp_status (0 = ok) and gp_last_error() describes the last failure on that context.
 *  - Quantities are exact int64: CPU in millicores (Quantity.MilliValue), memory in bytes, GPU in
 *    units -- the int64 model of resource.Quantity (SURVEY App. A.4).  Inputs that are not
 *    representable that way must be routed by the caller to the original Go packer.
 *  - Nodes are addressed by index into the caller's node table; names never cross the boundary.
 *  - A gp_ctx is NOT thread-safe (one per calling goroutine role, or a mutex), owns one CUDA
 *    stream, and there is NO CPU fallback: if no CUDA device is usable gp_create fails.
 */
#ifndef GANGPACK_H
#define GANGPACK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GP_ABI_VERSION 1

typedef struct gp_ctx gp_ctx;

typedef enum {
    GP_OK = 0,
    GP_ERR_INVALID = 1,       /* bad argument / precondition (negative request, index out of range, duplicate in an order ...) */
    GP_ERR_CUDA = 2,          /* CUDA runtime error; message in gp_last_error */
    GP_ERR_NO_DEVICE = 3,     /* no usable sm_90 device: the library has no CPU path */
    GP_ERR_NO_SNAPSHOT = 4,   /* gp_pack_* before gp_set_snapshot */
    GP_ERR_CAPACITY = 5,      /* result buffer too small */
    GP_ERR_UNREPRESENTABLE = 6 /* quantity outside the exact-int64 domain (|v| >= 2^61) */
} gp_status;

/* binpack algorithm: the `binpack:` config values of internal/binpacker/binpack.go:21-24 */
typedef enum {
    GP_TIGHTLY_PACK = 0,      /* "tightly-pack"      -> pack_tightly.go:34-63, ExecutorNodes node-major  */
    GP_DISTRIBUTE_EVENLY = 1, /* "distribute-evenly" -> distribute_evenly.go:34-73, round-major (also the
                                 fallback for unknown names, binpack.go:52-57) */
    GP_MINIMAL_FRAGMENTATION = 2 /* binpack.MinimalFragmentation -> LIB/binpack/minimal_fragmentation.go:27-137 over
                                 LIB/capacity/capacity.go:36-113: as few nodes as possible, fullest-fitting node first;
                                 ExecutorNodes in (capacity descending, priority order) then the remainder's node.
                                 GP_MODE_INDEPENDENT only: the building block of "single-az-minimal-fragmentation"
                                 (internal/binpacker/binpack.go:48), which packs one application per zone (zone =
                                 instance group) and chooses the zone on the host */
} gp_algo;

typedef enum {
    /* every app is packed against the same unmodified snapshot: the shape of
       internal/extender/unschedulablepods.go:132-166 and of each Predicate's own pack (resource.go:321) */
    GP_MODE_INDEPENDENT = 0,
    /* fitEarlierDrivers (resource.go:224-262): apps in queue order per instance group against a
       MUTATING snapshot, usage charged like sparkResourceUsage (sparkpods.go:139-146: each distinct
       executor node one executor; a driver node that hosts an executor is charged the executor only) */
    GP_MODE_FIFO_REFERENCE = 1,
    /* same loop with exact accounting (driver + every executor charged), i.e. what separate
       Predicate calls converge to through UsageForNodes (resources.go:31-43) */
    GP_MODE_FIFO_EXACT = 2
} gp_mode;

/* gp_config.flags */
#define GP_CFG_ASYNC_SNAPSHOT 1  /* gp_set_snapshot with page-locked (gp_alloc_pinned / gp_register_host) inputs returns while the
                                    device is still reading them: the buffers must stay unchanged until the next gp_pack_* /
                                    gp_get_snapshot / gp_synchronize call on the context has returned.  The upload then overlaps the
                                    input copies of that call (one Predicate = snapshot + pack, back to back).
                                    Also: a gp_pack_batch_device that directly follows gp_set_snapshot_device on the same stream
                                    (no other call on the context in between) may start before the slot layout has ended, so
                                    its inputs (application columns, offsets) must be ready before gp_set_snapshot_device is
                                    enqueued: a caller's kernel that writes them between the two calls would race with it */
typedef struct {
    int32_t device;          /* CUDA device ordinal; -1 = current device */
    int32_t flags;           /* GP_CFG_* */
    int32_t reserved[6];
} gp_config;

/* The node snapshot (NodeGroupSchedulingMetadata.AvailableResources, resources.go:61-100) plus the
 * two priority orders of NodeSorter.PotentialNodes (internal/sort/nodesorting.go:41-64), per
 * instance group.  Group g owns exec_order[exec_off[g]..exec_off[g+1]) and
 * drv_order[drv_off[g]..drv_off[g+1]); entries are indices into the node table, without
 * duplicates inside a group.  A driver candidate need not be an executor candidate.
 * Names absent from the metadata map are simply omitted by the caller (binpack.go:68-69,
 * pack_tightly.go:51-52: they can neither host a driver nor an executor). */
typedef struct {
    int32_t n_nodes;
    const int64_t* avail_cpu_milli;  /* [n_nodes] may be negative (over-committed node) */
    const int64_t* avail_mem_bytes;  /* [n_nodes] */
    const int64_t* avail_gpu;        /* [n_nodes] or NULL (= all zero) */
    int32_t n_groups;                /* >= 1 */
    const int32_t* exec_off;         /* [n_groups+1] */
    const int32_t* exec_order;       /* [exec_off[n_groups]] */
    const int32_t* drv_off;          /* [n_groups+1] */
    const int32_t* drv_order;        /* [drv_off[n_groups]] */
} gp_nodes;

/* The pending-application queue (types.SparkApplicationResources, internal/types/types.go:22-27, as
 * produced by sparkResources, internal/extender/sparkpods.go:73-137): SoA, queue order = index
 * order (creation-time ascending, sparkpods.go:67-69).  All requests must be >= 0. */
typedef struct {
    int32_t n_apps;
    const int64_t* drv_cpu_milli;    /* [n_apps] driver resources */
    const int64_t* drv_mem_bytes;
    const int64_t* drv_gpu;          /* or NULL (= 0) */
    const int64_t* exe_cpu_milli;    /* [n_apps] per-executor resources */
    const int64_t* exe_mem_bytes;
    const int64_t* exe_gpu;          /* or NULL (= 0) */
    const int32_t* exe_count;        /* [n_apps] MinExecutorCount (resource.go:242,325); >= 0, <= 2^24 (<= 2^20 in the
                                        FIFO modes); larger -> GP_ERR_UNREPRESENTABLE */
    const int32_t* group;            /* [n_apps] instance group, or NULL (= 0) */
    const uint8_t* skip_if_no_fit;   /* [n_apps] FIFO only: shouldSkipDriverFifo (resource.go:264-270), or NULL */
    const int64_t* exec_out_off;     /* [n_apps+1] exclusive prefix sum of exe_count, or NULL (computed) */
} gp_apps;

/* binpack.PackingResult (binpack.go:25-30) for a batch.
 *   driver_node[i] >= 0 : HasCapacity, DriverNode = that node index
 *                  == -1: HasCapacity=false (EmptyPackingResult)
 *                  == -2: not evaluated -- an earlier app of its group blocked the FIFO queue
 *   executor_nodes[exec_out_off[i] .. +exe_count[i]) : ExecutorNodes, in the reference's order
 *     (reservation names executor-1..k follow it, resourcereservations.go:501-510); its contents are
 *     UNDEFINED unless driver_node[i] >= 0 (the FIFO kernels emit optimistically before feasibility is known).
 * The per-node PackingEfficiencies map is not returned; its cluster-wide average, the Predicate's metric, is
 * gp_packing_efficiency (SURVEY §8a A7). */
typedef struct {
    int32_t* driver_node;            /* [n_apps] */
    int32_t* executor_nodes;         /* [executor_nodes_cap] */
    int64_t executor_nodes_cap;      /* entries available; must be >= sum(exe_count) */
} gp_results;

/* ---- lifecycle ------------------------------------------------------------------------- */
int gp_abi_version(void);
gp_status gp_create(gp_ctx** out, const gp_config* cfg /* may be NULL */);
void gp_destroy(gp_ctx* ctx);
const char* gp_last_error(const gp_ctx* ctx /* NULL = creation errors */);
/* 1 = CUDA (the only backend).  Present so a shim can assert it is not on a silent fallback. */
int gp_backend(const gp_ctx* ctx);

/* Pinned host memory for the SoA buffers that cross the boundary (cudaHostAlloc); a Go caller
 * wraps it with unsafe.Slice.  Pageable memory is accepted everywhere, just slower. */
gp_status gp_alloc_pinned(gp_ctx* ctx, size_t bytes, void** out);
gp_status gp_free_pinned(gp_ctx* ctx, void* p);

/* Page-locks caller-owned host memory (cudaHostRegister, portable + mapped) so that gp_pack_batch can DMA results
 * straight into it / read inputs in place -- e.g. a POSIX shared-memory segment that the scheduler process and the
 * per-GPU worker processes of one box share: every worker copies its block of the placements over its OWN PCIe
 * link into the scheduler's buffer (no gather through one GPU).  The range must stay mapped until unregistered. */
gp_status gp_register_host(gp_ctx* ctx, void* p, size_t bytes);
gp_status gp_unregister_host(gp_ctx* ctx, void* p);

/* ---- snapshot ------------------------------------------------------------------------------ */
/* Validates, copies to the device and lays the snapshot out in executor-priority order. */
gp_status gp_set_snapshot(gp_ctx* ctx, const gp_nodes* nodes);
/* Current device snapshot back in node-table order (after FIFO modes: with the usage subtracted,
 * i.e. metadata after SubtractUsageIfExists, resources.go:129-135).  Any pointer may be NULL. */
gp_status gp_get_snapshot(gp_ctx* ctx, int64_t* avail_cpu_milli, int64_t* avail_mem_bytes, int64_t* avail_gpu);

/* ---- availability snapshot from reservations (SURVEY 8f row f2) ------------------------------ */
/* GetReservedResources (internal/extender/resourcereservations.go:258-263: UsageForNodes over the hard
 * reservations, LIB/resources/resources.go:31-43, plus the soft reservations, internal/cache/
 * softreservations.go:155-170) followed by NodeSchedulingMetadataForNodes (resources.go:61-100):
 *   available[n]   = allocatable[n] - (sum of reservations on n + overhead[n])
 *   schedulable[n] = allocatable[n] - overhead[n]
 * One entry of res_* per reservation (hard and soft alike); res_node = index into the node table, or -1 for a
 * reservation whose node is not in the table (ignored, like the map lookup at resources.go:72-75; any index outside
 * [0, n_nodes) is treated so).
 *
 * Domain.  The reference's quantities have no bound; this library computes in the exact-int64 domain |v| < 2^61, and every
 * entry that takes a gp_usage_input (gp_build_availability, gp_build_reschedule_availability, gp_prepare_cluster,
 * gp_prepare_cluster_zones, gp_reschedule_from_reservations, gp_reconcile_find_nodes) returns either the exact result or
 * GP_ERR_UNREPRESENTABLE, never a wrapped one.  Refused: |allocatable|, |overhead| or a counted |reservation| >= 2^61; a
 * node whose reservations add up, exactly, to a sum outside the domain (the sum is not taken modulo 2^64: reservations that
 * add up to 2^64 are refused, not read as 0); an available, schedulable or -- where the entry computes it -- first-fit
 * availability outside the domain, or gp_reschedule_from_reservations' availability - overhead of the minimal-fragmentation
 * branch.  n_reservations >= 2^31 is GP_ERR_INVALID.  A refused call writes none of its outputs, except that
 * gp_reschedule_from_reservations and gp_reconcile_find_nodes leave theirs undefined, and it replaces nothing in the
 * context: after a refused gp_prepare_cluster or gp_prepare_cluster_zones the snapshot, layout, schedulable resources and
 * held az-aware orders are those of the last successful call (both synchronise the stream once, after the sort, to know). */
typedef struct {
    int32_t n_nodes;
    const int64_t* alloc_cpu_milli;      /* [n_nodes] node.Status.Allocatable */
    const int64_t* alloc_mem_bytes;
    const int64_t* alloc_gpu;            /* or NULL (= 0) */
    const int64_t* overhead_cpu_milli;   /* [n_nodes] OverheadComputer.GetOverhead, or NULL (= 0) */
    const int64_t* overhead_mem_bytes;   /* or NULL */
    const int64_t* overhead_gpu;         /* or NULL */
    int64_t n_reservations;
    const int32_t* res_node;             /* [n_reservations] */
    const int64_t* res_cpu_milli;
    const int64_t* res_mem_bytes;
    const int64_t* res_gpu;              /* or NULL (= 0) */
} gp_usage_input;
/* Outputs are [n_nodes] each; any of them may be NULL. */
gp_status gp_build_availability(gp_ctx* ctx, const gp_usage_input* in,
                                int64_t* avail_cpu_milli, int64_t* avail_mem_bytes, int64_t* avail_gpu,
                                int64_t* sched_cpu_milli, int64_t* sched_mem_bytes, int64_t* sched_gpu);

/* availableResources of rescheduleExecutor's FIRST-FIT branch (internal/extender/resource.go:638-643), bug for bug: the
 * reference calls NodeSchedulingMetadataForNodes(availableNodes, usage, overhead) -- which adds the overhead into the usage
 * map's EXISTING entries in place (resources.go:72-76) -- and then usage.Add(overhead) once more, so
 *   available[n] = allocatable[n] - (sum of reservations on n + overhead[n] * (n carries a reservation ? 2 : 1))
 * (SURVEY App. B7).  This is the availability to upload with gp_set_snapshot before gp_reschedule_executors(min_frag = 0);
 * the minimal-fragmentation branch uses the plain gp_build_availability output (:640, :682). */
gp_status gp_build_reschedule_availability(gp_ctx* ctx, const gp_usage_input* in,
                                           int64_t* avail_cpu_milli, int64_t* avail_mem_bytes, int64_t* avail_gpu);

/* ---- node priority order (the step before the hot path; SURVEY 8f row f1) ------------------- */
/* NodeSorter.PotentialNodes (internal/sort/nodesorting.go:41-64) on the device: nodes in ascending
 * (AZ priority, available memory, available CPU, name) order (:83-122), split into the driver candidates
 * (restricted to kube-scheduler's NodeNames, :52-54) and the executor candidates (schedulable && ready,
 * :55-57), each optionally re-sorted stably by the rank of a configured label value (:61-62,161-200).
 * The outputs are node indices and can be passed straight to gp_nodes.drv_order / exec_order.
 * Where the reference's comparators leave the order undefined (equal zone totals; equal (memory, cpu) with
 * different gpu, SURVEY App. B6) zones are ordered by id and nodes by name.
 * avail_* may hold any int64: keys are compared as signed 64-bit values, and the zone totals are summed and compared
 * exactly, beyond 64 bits where they get there (a zone id without nodes totals (0, 0) and takes its rank among all n_zones
 * ids like any other).  GP_ERR_INVALID: zone_id outside [0, n_zones), name_rank outside [0, n_nodes) or not a permutation
 * (a rank given twice) -- in every entry that takes a gp_sort_input. */
typedef struct {
    int32_t n_nodes;
    const int64_t* avail_cpu_milli;      /* [n_nodes] */
    const int64_t* avail_mem_bytes;      /* [n_nodes] */
    int32_t n_zones;                     /* >= 1 */
    const int32_t* zone_id;              /* [n_nodes] dense ids 0..n_zones-1 (ZoneLabel interned in first-seen order), or NULL (one zone) */
    const int32_t* name_rank;            /* [n_nodes] rank of the node name in ascending byte order: a permutation of 0..n_nodes-1
                                            (checked), or NULL (= index order) */
    const uint8_t* is_driver_candidate;  /* [n_nodes] member of ExtenderArgs.NodeNames, or NULL (= all) */
    const uint8_t* unschedulable;        /* [n_nodes] node.Spec.Unschedulable, or NULL (= none) */
    const uint8_t* ready;                /* [n_nodes] NodeReady == True, or NULL (= all) */
    const int32_t* driver_label_rank;    /* [n_nodes] rank of the node's value of driver-prioritized-node-label, -1 unknown; NULL = not configured */
    const int32_t* executor_label_rank;  /* same for executor-prioritized-node-label */
    const int64_t* avail_gpu;            /* [n_nodes] or NULL: only used to DETECT the ties below (gp_prepare_cluster: taken from the
                                            availability it computes) */
    int32_t* undefined_ties;             /* out, or NULL: number of adjacent pairs of the node order whose relative order the
                                            reference's comparator leaves undefined -- same zone priority, memory and cpu but
                                            different gpu (scheduleContextLessThan, nodesorting.go:83-93, is then "not less" both
                                            ways and sort.Slice is unstable; SURVEY App. B6).  Non-zero: this library ordered them
                                            by name; a shim that wants the reference's own (unspecified) choice falls back to Go */
} gp_sort_input;
gp_status gp_potential_nodes(gp_ctx* ctx, const gp_sort_input* in,
                             int32_t* driver_order /* [n_nodes] */, int32_t* n_driver,
                             int32_t* executor_order /* [n_nodes] */, int32_t* n_executor);

/* ---- everything before the hot path in one call ---------------------------------------------- */
/* gp_build_availability -> gp_potential_nodes -> gp_set_snapshot chained on the device: the availability computed
 * from the reservations never returns to the host, the two priority orders are consumed where they are produced
 * and the context ends up with a one-group snapshot ready for gp_pack_batch (what selectDriverNode does at
 * internal/extender/resource.go:300-304 before the FIFO loop).  sort->avail_* are ignored.  Node indices in later
 * results refer to this node table. */
gp_status gp_prepare_cluster(gp_ctx* ctx, const gp_usage_input* usage, const gp_sort_input* sort,
                             int32_t* n_driver /* may be NULL */, int32_t* n_executor /* may be NULL */);

/* gp_prepare_cluster for every instance group at once: the snapshot gp_pack_batch drains one FIFO queue per instance group
 * from (tightly-pack, distribute-evenly; apps->group = the instance group), built on the device.
 *   instance_group  [n_nodes] as in gp_prepare_cluster_zones_groups: in [0, n_instance_groups), -1 = in none, NULL = every node
 *                   in instance group 0.  Instance groups are disjoint node sets.  A node in none is in no order, but its
 *                   availability is computed and gp_get_snapshot returns it.
 *   availability    computed once for every node, exactly as gp_prepare_cluster computes it, with the same domain and
 *                   GP_ERR_UNREPRESENTABLE refusal.
 *   snapshot group i = instance group i: its driver and executor orders are PotentialNodes over i's nodes alone -- zone
 *                   priority from i's own (instance group, zone) exact totals, the candidate / schedulable / ready filters, the
 *                   stable label re-sort within i, the undefined-tie rule.
 * Identity: instance group i's orders, counts and undefined ties equal gp_prepare_cluster + gp_potential_nodes on a node table
 * holding only i's nodes (with their reservations), node indices mapped back to this table; an instance group without nodes
 * gets empty orders.  With instance_group == NULL or n_instance_groups == 1 (every node in 0) the context is exactly as after
 * gp_prepare_cluster.  sort->undefined_ties (if given) is the total.
 * SchedulableResources are kept as after gp_prepare_cluster.  The context is then ready for gp_pack_batch /
 * gp_pack_batch_device in every mode, gp_reserve_placements, gp_apply_usage_delta and gp_packing_efficiency[_groups]; the
 * snapshot survives FIFO calls, gp_reserve_placements and gp_apply_usage_delta.  A held zone layout is cleared, so the zone
 * entries' orders == NULL / groups == NULL forms are refused afterwards.
 * GP_ERR_INVALID (gp_last_error names the cause): what gp_prepare_cluster refuses; n_instance_groups < 1; an instance_group value
 * outside [-1, n_instance_groups); n_instance_groups > 1 with n_instance_groups x (sort->n_zones + 1) above 2^22 (the
 * per-(instance group, zone) zone totals).  A refused call replaces nothing (one synchronise after the availability stage, as
 * gp_prepare_cluster).  One synchronise more for the counts and undefined_ties; the four order arrays cost one more copy. */
typedef struct {
    int32_t n_driver;            /* out: driver candidates over every instance group */
    int32_t n_executor;          /* out: executor candidates over every instance group */
    int32_t* exec_off;           /* out, or NULL: [n_instance_groups + 1] CSR of exec_order (= the snapshot's exec_off) */
    int32_t* exec_order;         /* out, or NULL: [n_nodes] executor orders, instance group by instance group */
    int32_t* drv_off;            /* out, or NULL: [n_instance_groups + 1] CSR of drv_order (= the snapshot's drv_off) */
    int32_t* drv_order;          /* out, or NULL: [n_nodes] driver orders */
    int32_t* undefined_ties;     /* out, or NULL: [n_instance_groups] undefined ties of each instance group's order */
} gp_instance_group_orders;
gp_status gp_prepare_cluster_groups(gp_ctx* ctx, const gp_usage_input* usage, const gp_sort_input* sort,
                                    const int32_t* instance_group /* [n_nodes], or NULL = every node in group 0 */,
                                    int32_t n_instance_groups, gp_instance_group_orders* out);

/* The same chain for the zone-aware packers (SURVEY 8f rows f1/f2/f3): gp_prepare_cluster's availability and priority orders
 * (label re-sort and undefined_ties included), then both orders grouped by sort->zone_id on the device -- groupNodesByZone
 * (LIB/binpack/single_az.go:57-73).  Candidate zones have at least one driver and one executor candidate (:36-41); they are
 * ordered by the first position at which each appears in the driver order AFTER the label re-sort (driverZonesInOrder), and
 * each group's orders are the undivided orders restricted to that zone.  zone_id NULL or n_zones == 1: one zone.
 *   GP_LAYOUT_SINGLE_AZ  the groups are the candidate zones, every other node is dropped; no candidate zone = ONE empty group
 *                        (every gp_pack_*_zones result is then zone -1, the EmptyPackingResult of :31-33).  For
 *                        gp_pack_batch_zones / gp_pack_fifo_zones.
 *   GP_LAYOUT_AZ_AWARE   the candidate zones, then one trailing group with every other node of either order in undivided order
 *                        (present when non-empty or when no zone is a candidate): the layout of gp_pack_fifo_az_aware /
 *                        gp_pack_batch_az_aware, which then take orders == NULL to mean the undivided orders and n_zones this
 *                        call left on the device (az_aware_pack_tightly.go:27-38).
 * SchedulableResources (allocatable - overhead) are kept as if gp_set_schedulable had been called with them, and gp_get_snapshot
 * works as after gp_prepare_cluster.  The layout stays valid across FIFO calls, gp_reserve_placements and gp_apply_usage_delta
 * (they change availability, not orders); gp_set_snapshot, gp_set_snapshot_device, gp_prepare_cluster or another
 * gp_prepare_cluster_zones replaces it.  One stream synchronise for the counts; the optional arrays cost one more copy. */
typedef enum { GP_LAYOUT_SINGLE_AZ = 0, GP_LAYOUT_AZ_AWARE = 1 } gp_zone_layout_kind;
typedef struct {
    int32_t kind;              /* in: gp_zone_layout_kind */
    int32_t n_zones;           /* out: candidate zones = instance groups 0..n_zones-1, in driverZonesInOrder order */
    int32_t n_groups;          /* out: instance groups of the snapshot laid out */
    int32_t n_driver;          /* out: length of the undivided driver order (PotentialNodes' driverNodes) */
    int32_t n_executor;        /* out: length of the undivided executor order */
    int32_t reserved;
    int32_t* zone_of_group;    /* out, or NULL: [sort->n_zones + 1] zone id of each group, -1 = trailing / empty group */
    int32_t* exec_off;         /* out, or NULL: [n_groups + 1]   } the grouped layout as gp_nodes would carry it; */
    int32_t* exec_order;       /* out, or NULL: [n_nodes]        } copied back only when asked (logging, tests)  */
    int32_t* drv_off;          /* out, or NULL: [n_groups + 1] */
    int32_t* drv_order;        /* out, or NULL: [n_nodes] */
} gp_zone_layout;
gp_status gp_prepare_cluster_zones(gp_ctx* ctx, const gp_usage_input* usage, const gp_sort_input* sort, gp_zone_layout* layout);

/* gp_prepare_cluster_zones for every instance group at once: the snapshot gp_pack_fifo_zones_groups drains, built on the
 * device.  selectDriverNode ranks the nodes of ONE instance group (PotentialNodes over the affinity-filtered node set,
 * internal/extender/resource.go:292-304; zone priority over that set's zones only, internal/sort/nodesorting.go:95-121).
 *   instance_group  [n_nodes] the instance group of each node -- its instance-group-label value interned by the caller, or
 *                   the driver affinity of each instance group matched with gp_match_node_affinity -- in
 *                   [0, n_instance_groups), -1 = in none; NULL = every node in instance group 0.  Instance groups are
 *                   disjoint node sets.  A node in none is in no order, but its availability is computed and gp_get_snapshot
 *                   returns it.
 *   availability    computed once for every node, exactly as gp_prepare_cluster_zones computes it (GetReservedResources and
 *                   the overhead are per node, resource.go:300-303), with the same domain and GP_ERR_UNREPRESENTABLE refusal.
 *   per instance group i: the driver and executor orders are PotentialNodes over i's nodes alone -- zone priority from
 *                   per-(instance group, zone) exact totals, the candidate / schedulable / ready filters, the stable label
 *                   re-sort within i, the undefined-tie rule -- grouped by zone exactly as gp_prepare_cluster_zones groups
 *                   them (candidate zones in driverZonesInOrder order; GP_LAYOUT_SINGLE_AZ: they, or one empty group when
 *                   there is none; GP_LAYOUT_AZ_AWARE: plus the trailing group, LIB/binpack/single_az.go:36-41,57-73,
 *                   az_aware_pack_tightly.go:27-38).
 * Identity: instance group i's slice -- its groups group_off[i] .. group_off[i+1]-1, their zone_of_group, offsets and orders,
 * its undivided orders, n_zones[i] and undefined_ties[i] -- equals what gp_prepare_cluster_zones returns on a node table holding
 * only i's nodes (with their reservations), node indices mapped back to this table.  An instance group without nodes gets
 * the layout of "no candidate zone".  Instance groups are laid out in id order, so their groups are contiguous: the
 * two-level layout of gp_instance_groups.  sort->undefined_ties (if given) is the total.
 * The context then holds this layout: gp_pack_fifo_zones_groups(groups == NULL) drains every instance group's queue from it.
 * It survives FIFO calls, gp_reserve_placements and gp_apply_usage_delta like gp_prepare_cluster_zones' layout; any other
 * snapshot-setting call replaces it.  With n_instance_groups == 1 the context is also exactly as after
 * gp_prepare_cluster_zones; with more, gp_pack_fifo_zones, gp_pack_batch_zones and gp_pack_*_az_aware(orders == NULL) are
 * refused (they would treat every instance group's zones as one instance group's).
 * GP_ERR_INVALID (gp_last_error names the cause): what gp_prepare_cluster_zones refuses; n_instance_groups < 1; an
 * instance_group value outside [-1, n_instance_groups); n_instance_groups > 1 with n_instance_groups x (sort->n_zones + 1)
 * above 2^22 (the per-(instance group, zone) scratch).  A refused call replaces nothing (one synchronise after the
 * availability stage, as gp_prepare_cluster_zones).  One synchronise more for the counts and the per-instance-group words;
 * the optional arrays below other than group_off, n_zones, exec_off, drv_off and undefined_ties cost one more copy. */
typedef struct {
    int32_t kind;                /* in: gp_zone_layout_kind */
    int32_t n_groups;            /* out: snapshot groups over every instance group */
    int32_t n_driver;            /* out: driver candidates over every instance group */
    int32_t n_executor;          /* out: executor candidates over every instance group */
    int32_t* group_off;          /* out, or NULL: [n_instance_groups + 1] snapshot groups of each instance group */
    int32_t* n_zones;            /* out, or NULL: [n_instance_groups] its candidate zones (its first groups) */
    int32_t* exec_off;           /* out, or NULL: [n_instance_groups + 1] CSR of exec_order */
    int32_t* exec_order;         /* out, or NULL: [n_nodes] undivided executor orders, instance group by instance group */
    int32_t* drv_off;            /* out, or NULL: [n_instance_groups + 1] CSR of drv_order */
    int32_t* drv_order;          /* out, or NULL: [n_nodes] undivided driver orders */
    int32_t* group_exec_off;     /* out, or NULL: [n_groups + 1] } the grouped layout as gp_nodes would carry it */
    int32_t* group_exec_order;   /* out, or NULL: [n_nodes]      } */
    int32_t* group_drv_off;      /* out, or NULL: [n_groups + 1] */
    int32_t* group_drv_order;    /* out, or NULL: [n_nodes] */
    int32_t* zone_of_group;      /* out, or NULL: [n_groups] zone id of each group, -1 = trailing / empty group; n_groups <=
                                    n_instance_groups + min(n_nodes, n_instance_groups x sort->n_zones) */
    int32_t* undefined_ties;     /* out, or NULL: [n_instance_groups] undefined ties of each instance group's order */
} gp_instance_group_layout;
gp_status gp_prepare_cluster_zones_groups(gp_ctx* ctx, const gp_usage_input* usage, const gp_sort_input* sort,
                                          const int32_t* instance_group /* [n_nodes], or NULL = every node in group 0 */,
                                          int32_t n_instance_groups, gp_instance_group_layout* layout);

/* ---- executors without a usable reservation (the step after the hot path; SURVEY 8f row f4) --- */
/* rescheduleExecutor's node choice (internal/extender/resource.go:594-673) for a BATCH of executor pods, every
 * decision independent against the current snapshot (its executor priority orders and availabilities):
 *   min_frag == 0: the first node of the order the executor fits on (:657-662);
 *   min_frag != 0: rescheduleExecutorWithMinimalFragmentation (:675-705) -- capacities from
 *                  capacity.GetNodeCapacities (LIB/capacity/capacity.go:78-102) with `reserved_*` taken off each
 *                  node (the reference passes its overhead map there, :682); a node already hosting executors of
 *                  the same application wins, then the smallest capacity >= 1, then the order.
 * The caller uploads with gp_set_snapshot the availability the reference would use for that branch
 * (availableResources of :643 for first fit, availableNodesSchedulingMetadata of :640 for min_frag). */
typedef struct {
    int32_t n_execs;
    const int64_t* exe_cpu_milli;        /* [n_execs] */
    const int64_t* exe_mem_bytes;        /* [n_execs] */
    const int64_t* exe_gpu;              /* [n_execs] or NULL (= 0) */
    const int32_t* group;                /* [n_execs] instance group of the executor's application, or NULL (= 0) */
    int32_t min_frag;
    /* min_frag only: */
    const int64_t* reserved_cpu_milli;   /* [n_nodes] or NULL (= 0) */
    const int64_t* reserved_mem_bytes;   /* [n_nodes] (required when reserved_cpu_milli is given) */
    const int64_t* reserved_gpu;         /* [n_nodes] or NULL (= 0) */
    const int64_t* host_off;             /* [n_execs + 1] CSR offsets into host_nodes, or NULL (no application hosts anything yet) */
    const int32_t* host_nodes;           /* node indices already hosting executors of the same application
                                            (getNodesWithExecutorsBelongingToSameApp, :683) */
} gp_reschedule;
/* node_out[i] = node index, or -1 ("not enough capacity to reschedule the executor", :672) */
gp_status gp_reschedule_executors(gp_ctx* ctx, const gp_reschedule* in, int32_t* node_out /* [n_execs] */);

/* The whole of rescheduleExecutor (internal/extender/resource.go:594-673) minus pod and lister I/O, from the reservations to
 * the node choice in ONE device call, for a batch of executors decided independently against the same state.  The node table
 * is availableNodes (getNodes(nodeNames), :604) as gp_prepare_cluster takes it:
 *   scope       NULL or keep_topology_zone == -1: every node.  keep_topology_zone >= 0: filterNodesToZone (:463-478) first --
 *               only nodes whose topology_zone equals it are kept, and zone totals, availabilities and the executor order
 *               see only them.  A node with topology_zone == -1 (label missing) is GP_ERR_INVALID, whatever its zone, as in
 *               the reference.  Choosing the zone (getCommonZoneForExecutorsApplication, :493-533) stays with the caller.
 *   order       the executor order PotentialNodes would build from the metadata availability alloc - (reservations + overhead):
 *               zone priority by (memory, cpu) totals over the kept nodes (equal totals by zone id; sort->zone_id is the
 *               sorter's zone, NodeSchedulingMetadata.ZoneLabel = failure-domain.beta.kubernetes.io/zone or "default",
 *               LIB/resources/resources.go:78-81 -- NOT the topology label of the scope, SURVEY App. B5), then (available memory,
 *               available cpu, name rank), schedulable && ready nodes only, stable label re-sort by executor_label_rank when
 *               given.  No sort runs: a node's position is the rank of its unique key, and each decision is an arg-min.
 *   first fit   (in->min_frag == 0, :657-662) the first node of that order with !GreaterThan against
 *               alloc - (reservations + overhead * (node carries a reservation ? 2 : 1)) -- gp_build_reschedule_availability.
 *   min-frag    (:675-705) capacities from the metadata availability with usage->overhead_* as "reserved" (:682); the hosting set
 *               is in->host_off / host_nodes in node-table indices (hosting nodes that are not kept executor candidates are
 *               ignored); a hosting node with capacity >= 1 wins, then the smallest capacity, then the order.
 *   node_out[i] = node-table index, or -1 ("not enough capacity", :672).
 *   ambiguous[i] = 1 when the reference's own choice is unspecified: another node qualifies equally well (first fit: it fits;
 *               min-frag: same hosting class and capacity) but scheduleContextLessThan (internal/sort/nodesorting.go:83-93)
 *               does not order it against the winner -- same label key, zone priority, memory and cpu, different gpu (SURVEY
 *               App. B6).  A shim that wants the reference's choice then falls back to Go.
 * sort->avail_*, is_driver_candidate, driver_label_rank and undefined_ties are ignored; in->reserved_* must be NULL and
 * in->group NULL or all 0.  The context's snapshot, schedulable resources, zone layout and held az-aware orders are left
 * untouched (the call has scratch of its own), so it may be interleaved with a resident driver snapshot.  Validation as in
 * gp_prepare_cluster and gp_reschedule_executors; one stream synchronise, at the end. */
typedef struct {
    int32_t keep_topology_zone;      /* -1: every node; >= 0: keep only nodes whose topology_zone equals it */
    int32_t reserved;
    const int32_t* topology_zone;    /* [n_nodes] id of the node's topology.kubernetes.io/zone label, -1 = label missing;
                                        required when keep_topology_zone >= 0 */
} gp_reschedule_scope;
gp_status gp_reschedule_from_reservations(gp_ctx* ctx, const gp_usage_input* usage, const gp_sort_input* sort,
                                          const gp_reschedule_scope* scope /* NULL = every node */,
                                          const gp_reschedule* in, int32_t* node_out /* [n_execs] */,
                                          uint8_t* ambiguous /* [n_execs] or NULL */);

/* ---- packing ------------------------------------------------------------------------------- */
/* One batch through the hot path with HOST buffers: H2D of the app SoA, kernels, D2H of the
 * results; returns when the results are in host memory.  FIFO modes mutate the device snapshot. */
gp_status gp_pack_batch(gp_ctx* ctx, const gp_apps* apps, gp_algo algo, gp_mode mode, gp_results* out);

/* ---- compact wire formats for the PCIe-bound host path ------------------------------------------------------------
 * The reference hands a packer six resource.Quantity values and a count per application (types.SparkApplicationResources,
 * internal/types/types.go:22-27) and reads ExecutorNodes back as strings (binpack.go:25-30); what crosses PCIe here is
 * chosen per batch by the shim:
 *   inputs   quantity_bits 64: int64 columns exactly as in gp_apps (60 B per application with offsets);
 *            quantity_bits 32: int32 columns -- millicores, (bytes >> mem_shift), gpu units -- 28 B per application.  Only
 *            when every value is exactly representable (memory a whole multiple of 2^mem_shift bytes, everything < 2^31);
 *            the library rebuilds the exact int64 quantities, so results are bit-identical to the 64-bit layout.
 *   offsets  exec_out_off NULL: the exclusive prefix sum of exe_count is derived on the device (the caller recomputes
 *            it with a running sum while it walks the results).
 *   results  node_bits 16: ExecutorNodes as uint16 node indices -- allowed when the node table has <= 65 535 entries;
 *            GP_MODE_INDEPENDENT with tightly-pack / distribute-evenly only (GP_ERR_INVALID otherwise). */
typedef struct {
    int32_t n_apps;
    int32_t quantity_bits;           /* 64 or 32 */
    int32_t mem_shift;               /* 32-bit layout only: 0..40 */
    int32_t reserved;
    const void* drv_cpu;             /* [n_apps] int64 or int32, as quantity_bits says */
    const void* drv_mem;
    const void* drv_gpu;             /* or NULL (= 0) */
    const void* exe_cpu;
    const void* exe_mem;
    const void* exe_gpu;             /* or NULL (= 0) */
    const int32_t* exe_count;        /* as in gp_apps */
    const int32_t* group;            /* or NULL */
    const uint8_t* skip_if_no_fit;   /* or NULL */
    const int64_t* exec_out_off;     /* [n_apps+1] or NULL (derived on the device) */
} gp_apps_wire;
typedef struct {
    int32_t* driver_node;            /* [n_apps] as in gp_results */
    void* executor_nodes;            /* int32[executor_nodes_cap] (node_bits 32) or uint16[executor_nodes_cap] (node_bits 16) */
    int64_t executor_nodes_cap;
    int32_t node_bits;               /* 32 or 16 */
    int32_t reserved;
} gp_results_wire;
gp_status gp_pack_batch_wire(gp_ctx* ctx, const gp_apps_wire* apps, gp_algo algo, gp_mode mode, gp_results_wire* out);

/* binpack.SparkBinPackFunction for one application (group 0 of the snapshot).
 * Returns GP_OK and *has_capacity; executor_nodes must hold exe_count entries. */
gp_status gp_pack_one(gp_ctx* ctx, gp_algo algo,
                      int64_t drv_cpu_milli, int64_t drv_mem_bytes, int64_t drv_gpu,
                      int64_t exe_cpu_milli, int64_t exe_mem_bytes, int64_t exe_gpu,
                      int32_t exe_count, int32_t* has_capacity, int32_t* driver_node, int32_t* executor_nodes);

/* ---- device-resident entry points (multi-GPU plumbing, kernel-only timing) ----------------- */
/* Same as gp_set_snapshot / gp_pack_batch but every array pointer inside gp_nodes / gp_apps /
 * gp_results is a DEVICE pointer on ctx's device (group, skip_if_no_fit and -- for independent tightly-pack /
 * distribute-evenly -- exec_out_off may be NULL) and nothing is copied or validated on the host.  Work is
 * enqueued on `stream` (a cudaStream_t; NULL = the context's stream) and NOT synchronised (the two
 * order lengths are passed by value so that no device->host read is needed).
 * gp_set_snapshot_device keeps no reference to the caller's arrays after it returns. */
gp_status gp_set_snapshot_device(gp_ctx* ctx, const gp_nodes* dev_nodes,
                                 int32_t n_exec_total /* = exec_off[n_groups] */,
                                 int32_t n_drv_total /* = drv_off[n_groups] */, void* stream);
gp_status gp_pack_batch_device(gp_ctx* ctx, const gp_apps* dev_apps, gp_algo algo, gp_mode mode,
                               gp_results* dev_out, void* stream);
/* the context's own stream (cudaStream_t) so callers can order their work / record events on it */
void* gp_stream(gp_ctx* ctx);
gp_status gp_synchronize(gp_ctx* ctx);

/* ---- single-AZ packers on the device (SURVEY 8f row f3) -----------------------------------------------------------
 * getSingleAZSparkBinFunction + chooseBestResult (LIB/binpack/single_az.go:23-97) for a BATCH of applications.  The
 * snapshot's instance groups are the candidate zones in driverZonesInOrder order (groupNodesByZone, :57-73; zones without
 * executor candidates are left out by the caller like :38-41).  Every application is packed in every zone
 * (algo GP_TIGHTLY_PACK = "single-az-tightly-pack", GP_MINIMAL_FRAGMENTATION = "single-az-minimal-fragmentation"), the
 * float64 packing efficiencies (LIB/binpack/efficiency.go:66-156) are evaluated in the reference's operation order --
 * [driver] + ExecutorNodes, duplicates kept, sequential sums, cpu through Quantity.Value() -- and the zone with the highest
 * AvgPackingEfficiency.Max wins: the first among equals, and none when every average is 0 (:80, :91).  For
 * minimal-fragmentation the efficiencies see the driver only (minimalFragmentation never adds its executors to
 * SparkBinPack's reserved map) -- kept.  "az-aware-tightly-pack" (az_aware_pack_tightly.go:27-38), which falls back to the
 * undivided orders when no zone wins, is gp_pack_batch_az_aware for independent decisions and gp_pack_fifo_az_aware under
 * FIFO (both below).
 * gp_set_schedulable: NodeSchedulingMetadata.SchedulableResources of the current snapshot's nodes (resources.go:61-100). */
gp_status gp_set_schedulable(gp_ctx* ctx, const int64_t* sched_cpu_milli, const int64_t* sched_mem_bytes, const int64_t* sched_gpu /* or NULL */);
typedef struct {
    int32_t* zone;                   /* [n_apps] chosen instance group (zone), -1 = EmptyPackingResult */
    int32_t* driver_node;            /* [n_apps] */
    int32_t* executor_nodes;         /* CSR by exec_out_off (or the prefix sum of exe_count); defined when zone >= 0 */
    int64_t executor_nodes_cap;
    double* avg_efficiency;          /* [n_apps][4] = AvgPackingEfficiency{CPU, Memory, GPU, Max} of the winner, or NULL */
} gp_zone_results;
gp_status gp_pack_batch_zones(gp_ctx* ctx, const gp_apps* apps /* group, skip_if_no_fit ignored */, gp_algo algo, gp_zone_results* out);
/* The FIFO loop with a single-AZ packer in ONE launch: fitEarlierDrivers (internal/extender/resource.go:224-262) when
 * binpacker.BinpackFunc is SingleAZTightlyPack / SingleAZMinimalFragmentation.  The applications are the queue in order;
 * each one is packed in every zone against the availability its predecessors left, the zone is chosen like above, the
 * winner's usage is subtracted (mode GP_MODE_FIFO_REFERENCE: sparkResourceUsage's map assignment, sparkpods.go:139-146;
 * GP_MODE_FIFO_EXACT: every pod) and the next application sees it.  An application that fits in no zone gets zone -1,
 * driver_node -1 and -- unless skip_if_no_fit[i] -- blocks the queue: everything behind it reports driver_node -2
 * (never evaluated, resource.go:244-253).  The availability the device holds afterwards is what the loop left (read it
 * with gp_get_snapshot).  At most 64 zones; exec_out_off must be NULL or the prefix sum of exe_count.
 * ("az-aware-tightly-pack" needs the undivided orders for its fallback: gp_pack_fifo_az_aware.) */
gp_status gp_pack_fifo_zones(gp_ctx* ctx, const gp_apps* apps /* group ignored */, gp_algo algo, gp_mode mode, gp_zone_results* out);

/* The FIFO loop with "az-aware-tightly-pack" (AzAwareTightlyPack, LIB/binpack/az_aware_pack_tightly.go:27-38) in ONE launch.
 * Each queued application is packed in every candidate zone with tightly-pack and the zone is chosen exactly like
 * gp_pack_fifo_zones; when no zone wins, SparkBinPack(tightlyPackExecutors) runs over the UNDIVIDED driver / executor orders
 * against the availability the loop holds at that point, on the device, before the next application is tried.  Either
 * placement is charged like gp_pack_fifo_zones (mode GP_MODE_FIFO_REFERENCE or GP_MODE_FIFO_EXACT); an application that
 * fits neither way blocks or is skipped like there.
 * Snapshot (gp_set_snapshot, then gp_set_schedulable): groups 0..n_zones-1 are the candidate zones in driverZonesInOrder
 * order (zones without executor candidates left out, single_az.go:38-41), each with the undivided orders restricted to its
 * nodes; groups n_zones.. hold the other nodes of the two orders (a zone with driver candidates only, executor candidates of
 * a zone without driver candidates), which only the fallback reaches.  With n_zones = 0 every application takes the
 * fallback: the loop is then plain FIFO tightly-pack.
 * Results as gp_pack_fifo_zones, plus: zone[i] == -1 && driver_node[i] >= 0 = the undivided fallback placed application i
 * (its avg_efficiency is four zeros: the reference does not use the fallback's efficiencies).
 * GP_ERR_INVALID (gp_last_error names the cause): an independent mode; n_zones above 64 or above n_groups; no
 * gp_set_schedulable; a snapshot from gp_set_snapshot_device / gp_prepare_cluster (no host copy to check the orders
 * against); order lengths other than exec_off[n_groups] / drv_off[n_groups]; an order entry out of range, repeated or not
 * listed by the snapshot in that role; a zone group whose order is not the undivided order restricted to its nodes.
 * orders == NULL: right after gp_prepare_cluster_zones(GP_LAYOUT_AZ_AWARE) only -- the undivided orders and n_zones that call
 * left on the device (more than 64 candidate zones: GP_ERR_INVALID as above); after any other snapshot GP_ERR_INVALID. */
typedef struct {
    int32_t n_zones;                 /* snapshot groups 0..n_zones-1 are the candidate zones (0..64 under FIFO, 0..n_groups
                                        for gp_pack_batch_az_aware) */
    int32_t n_exec;
    const int32_t* exec_order;       /* [n_exec] executorNodePriorityOrder, undivided, node indices */
    int32_t n_drv;
    const int32_t* drv_order;        /* [n_drv] driverNodePriorityOrder, undivided, node indices */
} gp_az_orders;
gp_status gp_pack_fifo_az_aware(gp_ctx* ctx, const gp_apps* apps /* group ignored */, gp_mode mode, const gp_az_orders* orders,
                                gp_zone_results* out);

/* "az-aware-tightly-pack" (AzAwareTightlyPack, LIB/binpack/az_aware_pack_tightly.go:27-38) for a batch of INDEPENDENT
 * decisions against the unmodified snapshot -- the Predicate's own pack (EXT/resource.go:321) with n_apps = 1, or the
 * unschedulable marker's many decisions (EXT/unschedulablepods.go:132-166).  Each application is packed in every candidate
 * zone with tightly-pack and the zone is chosen exactly like gp_pack_batch_zones; when no zone wins,
 * SparkBinPack(tightlyPackExecutors) runs over the UNDIVIDED orders.  Everything stays on the device: one stream
 * synchronise, at the end.  The device snapshot is not modified.
 * Snapshot and orders: the layout of gp_pack_fifo_az_aware (candidate zones in groups 0..n_zones-1, the other nodes of the
 * two orders in the groups after them, gp_set_schedulable required), with any n_zones from 0 to n_groups (no 64-zone
 * bound).  With n_zones = 0 the call is gp_pack_batch(GP_TIGHTLY_PACK, GP_MODE_INDEPENDENT) over the undivided orders.
 * Results: zone[i] >= 0 = that zone won, avg_efficiency its averages; zone[i] == -1 && driver_node[i] >= 0 = the fallback
 * placed application i (four zero averages); zone[i] == -1 && driver_node[i] == -1 = it fits nowhere.  exec_out_off may be
 * NULL or given, as in gp_pack_batch_zones; exe_count up to 2^24.
 * gp_stats: scan_path_apps = applications for which the fallback ran; nodes_scanned / drivers_tried include its scans.
 * GP_ERR_INVALID (gp_last_error names the cause): those of gp_pack_fifo_az_aware except the mode and the 64-zone bound
 * (n_zones negative or above n_groups).  orders == NULL as in gp_pack_fifo_az_aware, without the 64-zone bound. */
gp_status gp_pack_batch_az_aware(gp_ctx* ctx, const gp_apps* apps /* group, skip_if_no_fit ignored */, const gp_az_orders* orders,
                                 gp_zone_results* out);

/* ---- reservation table of a batch + a snapshot that stays on the device (SURVEY 8f rows f4 and f2) ---------------
 * gp_reserve_placements: newResourceReservation (internal/extender/resourcereservations.go:491-528) for every application
 * of a packed batch whose driver_node >= 0, as a flat SoA table the shim turns into ResourceReservation objects: one row
 * per reservation slot -- slot 0 = "driver", slot i = "executor-i" (executorReservationName, :530-533) -> node index and
 * the slot's resources; rows of one application are contiguous, applications in queue order.  With subtract_from_snapshot
 * != 0 the same kernel takes every reserved pod off the availability the device holds (exact accounting, what
 * UsageForNodes, LIB/resources/resources.go:31-43, adds up from these reservations on the next Predicate), so the next
 * gp_pack_* call needs no gp_set_snapshot.
 * gp_apply_usage_delta: reservations that appeared (sign = +1: availability goes down) or went away (sign = -1) since
 * the snapshot was laid out -- the incremental form of GetReservedResources (resourcereservations.go:258-263). */
typedef struct {
    int64_t rows_cap;                /* rows the arrays below can hold; sum over placed apps of 1 + exe_count */
    int32_t* app;                    /* [rows_cap] index of the application in the batch */
    int32_t* slot;                   /* 0 = "driver", i = "executor-i" */
    int32_t* node;                   /* Reservation.Node as node index */
    int64_t* cpu_milli;              /* Reservation.Resources */
    int64_t* mem_bytes;
    int64_t* gpu;                    /* or NULL (not returned) */
    int64_t n_rows;                  /* out */
} gp_reservation_table;
gp_status gp_reserve_placements(gp_ctx* ctx, const gp_apps* apps, const gp_results* placed /* host arrays of a previous gp_pack_batch */,
                                int32_t subtract_from_snapshot, gp_reservation_table* out /* may be NULL with subtract */);
gp_status gp_apply_usage_delta(gp_ctx* ctx, int64_t n_rows, const int32_t* node, const int64_t* cpu_milli, const int64_t* mem_bytes,
                               const int64_t* gpu /* or NULL */, int32_t sign /* +1 reserve, -1 release */);

/* ---- the Predicate's packing-efficiency metric (EXT/resource.go:329, 352) ---------------------------------------------
 * computeAvgPackingEfficiencyForResult (internal/extender/resource.go:372-381) of placed applications: ComputePackingEfficiencies
 * over EVERY node of the context's node table (LIB/binpack/efficiency.go:66-102, binpack.go:72-77) averaged like
 * ComputeAvgPackingEfficiency (:114-156), against the availability the device holds and the SchedulableResources of
 * gp_set_schedulable / gp_prepare_cluster / gp_prepare_cluster_zones.  avg_out[4*i..] = {CPU, Memory, GPU, Max}.
 * (internal/metrics/binpack.go:66 reports max(CPU, Memory) of it; that step stays with the caller.)
 *   placed     HOST gp_results as gp_pack_batch returns them: driver_node, executor_nodes in CSR by apps->exec_out_off (or the
 *              prefix sum of exe_count).  Zone results are wrapped: gp_results{zone_results.driver_node, .executor_nodes, cap}.
 *   reserved   per node, the driver plus every executor placed there (SparkBinPack's map, binpack.go:72-75 + pack_tightly.go:50:
 *              tightly-pack, distribute-evenly, the az-aware zone winner or its fallback); algo GP_MINIMAL_FRAGMENTATION (also
 *              for single-az-minimal-fragmentation winners): the driver only -- minimalFragmentation never adds its executors.
 *   charged    GP_MODE_INDEPENDENT: every row against the current device availability (what SparkBinPack saw for an
 *              independent batch on this snapshot).  GP_MODE_FIFO_REFERENCE / GP_MODE_FIFO_EXACT: n_apps must be 1 and that
 *              application's usage under that mode is already in the availability (the driver as the last entry of a FIFO
 *              call; gp_reserve_placements(subtract = 1) charges like FIFO_EXACT); it is added back first -- FIFO_REFERENCE:
 *              sparkResourceUsage's map (EXT/sparkpods.go:139-146: one executor per distinct executor node, a driver node
 *              that hosts an executor the executor only), FIFO_EXACT: every pod.
 *   driver_node[i] < 0: WorstAvgPackingEfficiency (four zeros).
 * Exact sums: the CPU, Memory and Max sums over every node and the GPU sum over the nodes whose schedulable GPU is non-zero are
 * each rounded ONCE, to nearest-even, from their exact real value (math.fsum of the reference's per-node terms; an empty or
 * all-zero sum is +0.0).  Then CPU, Memory and Max are divided by max(float64(n_nodes), 1) and GPU is gpuSum / nodesWithGPU, or
 * 1.0 when no node has GPUs.  The reference sums in Go map order, which changes from call to call; this result does not
 * depend on any order and lies within the recursive-summation bound of every order the reference can take.
 * Device availability, slots, zone layout, held az-aware orders and gp_last_stats are left untouched; one stream synchronise,
 * at the end.  GP_ERR_NO_SNAPSHOT: no snapshot.  GP_ERR_INVALID: no SchedulableResources, a node index out of range, a FIFO
 * charged mode with n_apps != 1, a negative request.  GP_ERR_CAPACITY: executor_nodes_cap too small.  GP_ERR_UNREPRESENTABLE:
 * a request, or a per-node reserved or added-back amount, >= 2^61. */
gp_status gp_packing_efficiency(gp_ctx* ctx, const gp_apps* apps, gp_algo algo, const gp_results* placed /* host */,
                                gp_mode charged, double* avg_out /* [n_apps][4] */);

/* gp_packing_efficiency averaged per instance group: the Predicate's metric as the reference computes it when a snapshot holds
 * several instance groups.  selectDriverNode builds its metadata from the nodes of the driver's instance group
 * (ListWithPredicate(driver affinity), EXT/resource.go:292-303), and ComputePackingEfficiencies runs over that metadata
 * (LIB/binpack/binpack.go:72-77, efficiency.go:66-156).  Row i is exactly gp_packing_efficiency's computation with "every node
 * of the table" replaced by {v : instance_group[v] == apps->group[i]} -- the per-node terms, the exact once-rounded sums, the
 * max(n, 1) divisor with n that instance group's node count, the nodesWithGPU rule, four zeros for driver_node < 0.
 *   instance_group  [n_nodes] in [0, n_instance_groups), -1 = in none (such a node counts in no row's average); instance
 *                   groups are disjoint.  Any snapshot works: gp_set_snapshot with several groups, gp_prepare_cluster_groups,
 *                   gp_prepare_cluster_zones_groups.
 *   apps->group     each row's instance group (NULL = 0).
 *   charged         as in gp_packing_efficiency, except that the FIFO modes allow at most ONE row per instance group (its
 *                   add-back then touches only its own instance group's nodes, and every row stays exact).
 * With n_instance_groups == 1 and every node in instance group 0 the result equals gp_packing_efficiency's, bit for bit.
 * Refusals: gp_packing_efficiency's, plus GP_ERR_INVALID for instance_group NULL (with nodes), n_instance_groups < 1, a value
 * outside [-1, n_instance_groups), a row's group outside [0, n_instance_groups), two rows of one instance group under a FIFO
 * charged mode, and a placed row whose driver or executor node lies outside its instance group.  One stream synchronise. */
gp_status gp_packing_efficiency_groups(gp_ctx* ctx, const gp_apps* apps /* group = instance group */, gp_algo algo,
                                       const gp_results* placed /* host */, gp_mode charged,
                                       const int32_t* instance_group /* [n_nodes] */, int32_t n_instance_groups,
                                       double* avg_out /* [n_apps][4] */);

/* ---- the Predicate's placement metrics (EXT/resource.go:352-357) ------------------------------------------------------------
 * What selectDriverNode reports about a successful pack besides the packing efficiency, for a batch of placed applications:
 * ReportInitialDriverExecutorCollocationMetric (internal/metrics/metrics.go:223-252), ReportInitialNodeCountMetrics (:254-275)
 * and ReportCrossZoneMetric with crossZoneTraffic (:277-318, 322-330).  Row i is one application: driver_node d,
 * ExecutorNodes e[0..k) (k = exe_count[i], in any order: node-major, round-major, capacity order or a zone result) and its
 * instance group.  The reference returns before these metrics when !HasCapacity (:347-350): a row with d < 0 (-1 and the FIFO
 * -2 alike) gets the "not reported" record {collocation -1, every other field 0}.  For d >= 0, with E the set of e:
 *   collocation          0 "no-collocation" when d is not in E (k = 0 included); 1 "driver-collocated-with-all-executors"
 *                        when d is in E and |E| = 1; 2 "driver-collocated-with-some-executors" otherwise.
 *   distinct_exec_nodes  |E|.
 *   execs_per_node       k / |E| with Go's integer division; -1 when k = 0 (ReportInitialNodeCountMetrics returns early).
 *   n_zones, cross_zone_pairs, total_pairs
 *                        pods per node: the driver's node 1, plus one per executor entry (a driver node that hosts executors
 *                        counts 1 + its executors); T = k + 1.  c_z = the pods on nodes of availableNodes whose metric zone is z;
 *                        pods on other nodes count in T and in no zone.  n_zones = #{z : c_z > 0}; total_pairs = T (T - 1) / 2;
 *                        cross_zone_pairs = T S - (S^2 + sum_z c_z^2) / 2 with S = sum_z c_z (exact: the numerator is even),
 *                        which is crossZoneTraffic for every iteration order of its map (DESIGN.md §2.8).  With k <= 2^24 (the
 *                        gp_apps bound) every value fits in int64.
 *   metric_zone          [n_nodes] the node's zone as the metric reads it, interned to 0..n_metric_zones-1: the label
 *                        failure-domain.beta.kubernetes.io/zone (v1.LabelZoneFailureDomain, :290) with a missing label
 *                        interned as the string "unknown-zone" -- so it merges with a node literally labelled unknown-zone.
 *                        NodeSchedulingMetadata.ZoneLabel reads the same key but maps a missing label to "default"
 *                        (LIB/resources/resources.go:27, 78-81), and the single-AZ packers and rescheduling read
 *                        topology.kubernetes.io/zone: none of their zone columns can be passed here as is.
 *   instance_group       [n_nodes] or NULL.  availableNodes is the driver's instance group (ListWithPredicate(driver affinity),
 *                        EXT/resource.go:292-295): node v is in row i's scope when instance_group[v] == apps->group[i] (NULL
 *                        group = 0), -1 = in no instance group.  NULL: every node of the table is in scope (the one-group
 *                        Predicate; apps->group and n_instance_groups are ignored).  A placed node outside the scope is allowed.
 * Emitting the counters, histograms, gauges and Mean() stays with the caller.
 * The call is stateless: it needs no snapshot and leaves the device availability, slots, zone layout, held az-aware orders and
 * gp_last_stats untouched.  apps: exe_count, group and exec_out_off are read (NULL exec_out_off = the prefix sum of exe_count).
 * GP_ERR_INVALID (gp_last_error names the cause): NULL arrays or negative sizes; n_metric_zones above max(n_nodes, 1) (an
 * interned id comes from some node); a driver or executor node of a placed row
 * outside [0, n_nodes); a metric_zone value outside [0, n_metric_zones); with instance_group, n_instance_groups < 1, a value
 * outside [-1, n_instance_groups) or a row's group outside [0, n_instance_groups); a negative exe_count.  GP_ERR_CAPACITY: a
 * placed row's ExecutorNodes outside [0, executor_nodes_cap).  GP_ERR_UNREPRESENTABLE: an exe_count above 2^24.  A refused call
 * writes no record.  One stream synchronise. */
typedef struct {
    int32_t collocation;             /* -1 not reported, 0 / 1 / 2 as above */
    int32_t distinct_exec_nodes;
    int32_t execs_per_node;
    int32_t n_zones;
    int64_t cross_zone_pairs;
    int64_t total_pairs;
} gp_placement_record;
gp_status gp_placement_metrics(gp_ctx* ctx, const gp_apps* apps, const gp_results* placed /* host */, int32_t n_nodes,
                               const int32_t* metric_zone /* [n_nodes] */, int32_t n_metric_zones,
                               const int32_t* instance_group /* [n_nodes] or NULL */, int32_t n_instance_groups,
                               gp_placement_record* out /* [n_apps] */);
/* The same on device arrays, enqueued on `stream` (a cudaStream_t; NULL = the context's stream) with no synchronise and no
 * host copy, like gp_pack_batch_device, whose outputs (driver_node, executor_nodes, and the apps it read) it reads in place.
 * Every array pointer inside apps / placed, metric_zone, instance_group and out is a device pointer on ctx's device;
 * exec_out_off may be NULL (derived on the device).  The checks above run on the device: *dev_status (one device int32, or
 * NULL) receives GP_OK, GP_ERR_INVALID, GP_ERR_UNREPRESENTABLE or GP_ERR_CAPACITY once the work has run, and the records are meaningful only when it
 * is GP_OK.  Arguments that need no device data (NULL pointers, negative sizes) are refused at once.  The call's scratch
 * belongs to the context: the next gp_placement_metrics* call on it must be ordered after this one (same stream, or an
 * event). */
gp_status gp_placement_metrics_device(gp_ctx* ctx, const gp_apps* dev_apps, const gp_results* dev_placed, int32_t n_nodes,
                                      const int32_t* metric_zone, int32_t n_metric_zones, const int32_t* instance_group,
                                      int32_t n_instance_groups, gp_placement_record* dev_out, int32_t* dev_status, void* stream);

/* ---- the unschedulable-pod marker's capacity checks (EXT/unschedulablepods.go:93-166) ------------------------------------
 * DoesPodExceedClusterCapacity (:132-166) for a batch of stale drivers, under any `binpack:` value, in one call.  Each driver is
 * packed against the nodes of its affinity class with zero usage -- NodeSchedulingMetadataForNodes(nodes, zero usage, overhead)
 * (LIB/resources/resources.go:61-100), so available = schedulable = allocatable - overhead on every node, unschedulable and
 * not-ready nodes included -- and the affinity nodes in lister order as both priority orders; exceeds[i] = !HasCapacity.
 * The answer depends on neither that order nor any placement (DESIGN §2.2): no sort, no layout and no placement is computed.
 *   nodes       allocatable and GetNonSchedulableOverhead per node; zone_id = ZoneLabel (failure-domain.beta.kubernetes.io/zone,
 *               "default" when absent) interned to 0..n_zones-1, NULL = one zone (only the single-AZ packers look at it);
 *               node_group = the affinity class of each node (0..n_groups-1), -1 = in none, NULL = every node in class 0.
 *   drivers     gp_apps with group = the driver's affinity class, -1 = its required affinity matches every node, NULL = 0;
 *               exe_count any int32 >= 0 (no 2^24 bound); skip_if_no_fit and exec_out_off are ignored.
 *   An affinity class with no nodes gives exceeds = 1.
 * The call is stateless with respect to the context: the snapshot, SchedulableResources, the zone layout, the held az-aware
 * orders and gp_last_stats are left untouched; it has scratch of its own and synchronises the stream once, at the end.
 * GP_ERR_INVALID (gp_last_error names the cause): a negative request or exe_count, a group or zone id out of range, an unknown
 * packer, n_groups < 1.  GP_ERR_UNREPRESENTABLE: a request, |allocatable| or |overhead| >= 2^61.  The node table is
 * validated with n_apps == 0 too.  On an error exceeds is undefined. */
typedef enum {
    GP_BP_TIGHTLY_PACK = 0,                    /* "tightly-pack" */
    GP_BP_DISTRIBUTE_EVENLY = 1,               /* "distribute-evenly" */
    GP_BP_AZ_AWARE_TIGHTLY_PACK = 2,           /* "az-aware-tightly-pack" */
    GP_BP_SINGLE_AZ_TIGHTLY_PACK = 3,          /* "single-az-tightly-pack" */
    GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION = 4  /* "single-az-minimal-fragmentation" */
} gp_binpacker;
typedef struct {
    int32_t n_nodes;
    const int64_t* alloc_cpu_milli;      /* [n_nodes] node.Status.Allocatable */
    const int64_t* alloc_mem_bytes;
    const int64_t* alloc_gpu;            /* or NULL (= 0) */
    const int64_t* overhead_cpu_milli;   /* [n_nodes] GetNonSchedulableOverhead, or NULL (= 0) */
    const int64_t* overhead_mem_bytes;   /* or NULL */
    const int64_t* overhead_gpu;         /* or NULL */
    int32_t n_zones;                     /* >= 1 when zone_id is given */
    const int32_t* zone_id;              /* [n_nodes] or NULL (one zone) */
    int32_t n_groups;                    /* >= 1 */
    const int32_t* node_group;           /* [n_nodes] affinity class, -1 = none; or NULL (all 0) */
} gp_capacity_nodes;
gp_status gp_exceeds_cluster_capacity(gp_ctx* ctx, const gp_capacity_nodes* nodes, const gp_apps* drivers, gp_binpacker packer,
                                      uint8_t* exceeds /* [n_apps] */);

/* ---- the FIFO loop of every instance group with a zone-aware packer, in ONE launch ---------------------------------------
 * fitEarlierDrivers (internal/extender/resource.go:224-262) walks one instance group's queue against that group's nodes
 * (resource.go:292-295); queues of different instance groups are independent.  gp_pack_fifo_zones_groups runs all of them at
 * once, one CTA per instance group, with packer GP_BP_SINGLE_AZ_TIGHTLY_PACK / GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION (as
 * gp_pack_fifo_zones) or GP_BP_AZ_AWARE_TIGHTLY_PACK (as gp_pack_fifo_az_aware), mode GP_MODE_FIFO_REFERENCE or
 * GP_MODE_FIFO_EXACT.
 * Snapshot (gp_set_snapshot, then gp_set_schedulable): the groups of instance group i are group_off[i] .. group_off[i+1]-1,
 * laid out for its packer as gp_pack_fifo_zones / gp_pack_fifo_az_aware expect them (single-AZ: every one a candidate zone,
 * at most 64; az-aware: the first n_zones[i] (at most 64) its candidate zones, the rest its trailing group, exec_order /
 * drv_order its undivided orders in CSR by exec_off / drv_off).  The queue of instance group i is the applications j with
 * apps->group[j] == i (group NULL: every application in instance group 0), in index order; skip_if_no_fit as there.
 * For every instance group each output -- zone (local to the instance group: 0 = its first candidate zone), driver_node
 * (-1 / -2 included: a blocked queue blocks its own instance group only), ExecutorNodes, avg_efficiency and the availability
 * left behind -- is what gp_pack_fifo_zones / gp_pack_fifo_az_aware return on a context holding only that instance group's
 * groups and applications.  gp_stats sums over the instance groups (scan_path_apps: the az-aware fallbacks).
 * GP_ERR_INVALID (gp_last_error names the cause; a refused call changes nothing): another packer or mode; no
 * gp_set_schedulable; explicit groups on a snapshot from gp_set_snapshot_device / gp_prepare_cluster* (no host copy of the layout); group_off
 * not monotone from 0 to the snapshot's n_groups; an application's group outside [0, n_instance_groups); more than 64
 * candidate zones in an instance group, or n_zones[i] above its group count; az-aware orders missing, with offsets not
 * monotone from 0 to the snapshot's executor / driver candidate counts, listing a node out of range, twice, of another
 * instance group or not in that role, or a zone group whose order is not its instance group's order restricted to it.
 * groups == NULL: the layout gp_prepare_cluster_zones_groups left on the context (its per-instance-group words kept on the
 * host, its undivided orders read on the device, no order check: the library built them).  Refused (GP_ERR_INVALID) after
 * any other snapshot-setting call (gp_set_snapshot, gp_set_snapshot_device, gp_prepare_cluster, gp_prepare_cluster_zones),
 * with a packer that does not match the layout's kind (single-AZ packers: GP_LAYOUT_SINGLE_AZ; az-aware:
 * GP_LAYOUT_AZ_AWARE), and with more than 64 candidate zones in an instance group. */
typedef struct {
    int32_t n_instance_groups;
    const int32_t* group_off;        /* [n_instance_groups + 1] snapshot groups of each instance group */
    const int32_t* n_zones;          /* az-aware: [n_instance_groups] candidate zones of each; NULL for the single-AZ packers */
    const int32_t* exec_off;         /* az-aware: [n_instance_groups + 1] CSR of exec_order; else NULL */
    const int32_t* exec_order;       /* az-aware: executorNodePriorityOrder of each instance group, undivided, node indices */
    const int32_t* drv_off;          /* az-aware: [n_instance_groups + 1] CSR of drv_order; else NULL */
    const int32_t* drv_order;        /* az-aware: driverNodePriorityOrder of each instance group, undivided, node indices */
} gp_instance_groups;
gp_status gp_pack_fifo_zones_groups(gp_ctx* ctx, const gp_apps* apps /* group = instance group */, gp_binpacker packer, gp_mode mode,
                                    const gp_instance_groups* groups, gp_zone_results* out);

/* ---- required node affinity (K8S = vendor/k8s.io) ------------------------------------------------------------------------
 * GetRequiredNodeAffinity(pod).Match(node) (K8S/component-helpers/scheduling/corev1/nodeaffinity/nodeaffinity.go:297-324) for
 * every (distinct affinity, node), as utils.ListWithPredicate runs it in selectDriverNode (EXT/resource.go:292-298) and in
 * DoesPodExceedClusterCapacity (EXT/unschedulablepods.go:133-139).  Outcome per node: match, no match or error:
 *   1. nodeSelector: every (key, value) must be a label of the node, else no match (even when the terms would have errored);
 *   2. no requiredDuringScheduling...: match;
 *   3. terms in order (nodeaffinity.go:56-103, 152-201): a term with a parse error records an error and is skipped, a term
 *      without requirements is skipped, a term matches when all its label and field requirements match; the first match wins;
 *   4. no term matched: no match, an error when a term recorded one.  A required affinity whose terms are all empty matches
 *      no node.
 * Label requirements (K8S/apimachinery/pkg/labels/selector.go:218-262): In = key present and value in the set; NotIn = key
 * absent or value not in the set; Exists / DoesNotExist = presence; Gt / Lt = key present, its value parses
 * (strconv.ParseInt(v, 10, 64)) and is strictly greater / less than the bound -- a value that does not parse is no match.
 * Field requirements: metadata.name In / NotIn one value, given as a node index (-1: no node has that name).  A field key other
 * than metadata.name reads "" (extractNodeFields sets no other field): the caller encodes In "" / NotIn v != "" as NotIn -1
 * (always true) and In v != "" / NotIn "" as In -1 (never true).
 * Strings never cross the boundary: the caller interns label keys and values to dense ids, and does what needs the strings --
 * NewRequirement's validation (an operator that is not one of the six, a key that is not a qualified name, a value that is not
 * a label value, In / NotIn without values, Exists / DoesNotExist with values, Gt / Lt without exactly one integer value;
 * matchFields other than In / NotIn with exactly one value) becomes the term's parse_error flag, ParseInt of a node's label value
 * becomes label_int_ok / label_int, metadata.name becomes a node index. */
typedef enum {
    GP_AFF_IN = 0, GP_AFF_NOT_IN = 1, GP_AFF_EXISTS = 2, GP_AFF_DOES_NOT_EXIST = 3, GP_AFF_GT = 4, GP_AFF_LT = 5,
    GP_AFF_FIELD_NAME_IN = 6, GP_AFF_FIELD_NAME_NOT_IN = 7
} gp_aff_op;
typedef struct {
    int32_t n_nodes;
    int32_t n_keys;                      /* label key ids 0..n_keys-1 */
    int32_t n_values;                    /* label value ids 0..n_values-1 */
    int32_t reserved;
    const int64_t* label_off;            /* [n_nodes+1] CSR: node i's labels are [label_off[i], label_off[i+1]); label_off[0] = 0 */
    const int32_t* label_key;            /* strictly ascending within a node (node.Labels is a map) */
    const int32_t* label_val;
    const uint8_t* label_int_ok;         /* ParseInt(value, 10, 64) succeeded; or NULL (no value parses) */
    const int64_t* label_int;            /* its result where label_int_ok; or NULL with label_int_ok */
} gp_node_labels;
typedef struct {
    int32_t n_aff;                       /* distinct required affinities (nodeSelector + requiredDuringScheduling...) */
    int32_t reserved;
    const int64_t* sel_off;              /* [n_aff+1] nodeSelector of affinity a: [sel_off[a], sel_off[a+1]) */
    const int32_t* sel_key;              /*   key id = value id, each */
    const int32_t* sel_val;
    const uint8_t* has_required;         /* [n_aff] requiredDuringScheduling... is not nil */
    const int64_t* term_off;             /* [n_aff+1] affinity a's terms, in order: [term_off[a], term_off[a+1]) */
    const int64_t* term_req_off;         /* [n_terms+1] term t's requirements: [term_req_off[t], term_req_off[t+1]) */
    const uint8_t* term_parse_error;     /* [n_terms] or NULL (none) */
    const int32_t* req_op;               /* [n_req] gp_aff_op */
    const int32_t* req_key;              /* [n_req] label key id (ignored by the field operators) */
    const int64_t* req_int;              /* [n_req] GT / LT: the bound; FIELD_NAME_*: node index or -1; else ignored */
    const int64_t* req_val_off;          /* [n_req+1] IN / NOT_IN value set: [req_val_off[r], req_val_off[r+1]) */
    const int32_t* req_val;              /*   value ids, strictly ascending within a requirement */
} gp_node_affinities;
typedef struct {
    uint32_t* member;                    /* [n_aff][(n_nodes+31)/32]: bit j%32 of word j/32 = node j matches; or NULL */
    int32_t* n_match;                    /* [n_aff] nodes that match; or NULL */
    int32_t* n_error;                    /* [n_aff] nodes whose outcome is an error (ListWithPredicate returns it: the
                                            Predicate fails with failureInternal); or NULL */
} gp_affinity_match;
/* The match of every affinity against every node, in one call.  An error node is not a member.
 * The context is left alone (snapshot, SchedulableResources, zone layout, held az-aware orders, gp_last_stats); scratch of its
 * own, one stream synchronise.  GP_ERR_INVALID (gp_last_error names the cause): missing arrays or negative sizes; offsets
 * that do not start at 0 or decrease; a label key or value id out of range; the keys of a node not strictly ascending; an
 * operator out of range; a selector or requirement key or value id out of range; a value set not strictly ascending; a field
 * node index outside [-1, n_nodes).  On an error the outputs are undefined. */
gp_status gp_match_node_affinity(gp_ctx* ctx, const gp_node_labels* labels, const gp_node_affinities* affinities,
                                 gp_affinity_match* out);

/* gp_exceeds_cluster_capacity with each driver's node set = the nodes its required affinity matches, evaluated in the same
 * call: any subsets of the nodes, overlapping freely (DoesPodExceedClusterCapacity, EXT/unschedulablepods.go:132-166).
 *   nodes       as for gp_exceeds_cluster_capacity, with node_group NULL and n_groups ignored; labels->n_nodes = nodes->n_nodes.
 *   drivers     group = the driver's affinity id, 0..n_aff-1 (required); exe_count any int32 >= 0.
 *   exceeds[i]  = !HasCapacity over driver i's matched nodes: the T + M criterion (DESIGN §2.2), per zone for the single-AZ
 *               packers; an empty match gives 1.
 *   affinity_error[i] = 1 when driver i's affinity gives an error on some node (ListWithPredicate fails: the marker's scan
 *               returns at that driver, unschedulablepods.go:113-117); exceeds[i] is then undefined.  May be NULL.
 * The scratch is bounded whatever the total membership: the affinities are processed in chunks. Context left alone, one
 * stream synchronise.  Refusals: those of both calls, and node_group not NULL, a driver group outside [0, n_aff). */
gp_status gp_exceeds_cluster_capacity_affinity(gp_ctx* ctx, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                                               const gp_node_affinities* affinities, const gp_apps* drivers, gp_binpacker packer,
                                               uint8_t* exceeds /* [n_apps] */, uint8_t* affinity_error /* [n_apps] or NULL */);

/* ---- the failover reconciler's node choice (EXT/failover.go:43-82, 286-436) ------------------------------------------------
 * syncResourceReservationsAndDemands minus pod, lister and CRD I/O: availableResourcesPerInstanceGroup (:286-323), then for each
 * stale driver in call order constructResourceReservation's findNodes (:348-390, 409-436) and the charge of :159, in one call.
 *   usage       the node table with every hard and soft reservation row and GetOverhead, exactly as gp_build_availability takes
 *               it: available = allocatable - (reservations + overhead).
 *   nodes       node_group = the interned value of the node's instanceGroupLabel ("" is a group like any other); creation orders
 *               like metav1.Time.Before (UnixNano); unschedulable / not-ready nodes belong to no group's order.  Each group's
 *               order is its schedulable, ready nodes by (creation descending, node-table index) -- the reference's newest-first
 *               sort.Slice when the lister returns the nodes in that order (DESIGN §2.3).
 *   stale       exe_cpu/mem/gpu, group (NULL = 0) and exe_count = max(0, MinExecutorCount - running executors) per driver, in the
 *               order the reservations are written; drv_* and skip_if_no_fit are ignored; exec_out_off NULL or the prefix sum.
 *   placed[i]   -1: the driver's group has no schedulable, ready node ("instance group not found", :358-362; nothing charged,
 *               even with exe_count 0); otherwise len(reservedNodeNames), 0..exe_count (less: the group ran out of room).
 *   executor_nodes[exec_out_off[i] ..) the reservedNodeNames as node indices, node-major; entries past placed[i] undefined.
 *   Each node the walk reaches is charged (t + 1) x exe when it took t executors and the walk went on, t x exe when it completed
 *   the driver there (DESIGN §2.3); the running driver and executors of a stale application are never charged.
 * The context is left alone: snapshot, SchedulableResources, zone layout, held az-aware orders and gp_last_stats stay as they
 * were; the call has scratch of its own and synchronises the stream once, at the end.
 * GP_ERR_INVALID: missing arrays, n_groups < 1, a node or driver group out of range, a negative request or exe_count, an
 * exec_out_off that is not the prefix sum.  GP_ERR_UNREPRESENTABLE: a request >= 2^61, exe_count > 2^24, or an availability the
 * loop reads or charges outside the exact-int64 domain (|v| >= 2^61; the reference's quantities have no bound, so repeated
 * overshoot charges can leave it) -- the whole call is refused, nothing wraps.  GP_ERR_CAPACITY: executor_nodes_cap too small.
 * On an error the outputs are undefined. */
typedef struct {
    int32_t n_groups;              /* instance-group ids 0..n_groups-1 (instanceGroupLabel values interned; "" included) */
    int32_t reserved;
    const int32_t* node_group;     /* [usage->n_nodes] */
    const int64_t* creation;       /* [n_nodes] ordered like metav1.Time.Before (UnixNano) */
    const uint8_t* unschedulable;  /* or NULL */
    const uint8_t* ready;          /* or NULL (= all) */
} gp_reconcile_nodes;
typedef struct {
    int32_t* placed;               /* [n_apps] len(reservedNodeNames), 0..exe_count; -1 = instance group not found */
    int32_t* executor_nodes;       /* node-major at exec_out_off[i]; entries past placed[i] undefined */
    int64_t executor_nodes_cap;
    int64_t* avail_cpu_milli;      /* out or NULL: [n_nodes] availability after the loop (the only direct */
    int64_t* avail_mem_bytes;      /*   observable of the overshoot charge; tests and logging)            */
    int64_t* avail_gpu;
} gp_reconcile_results;
gp_status gp_reconcile_find_nodes(gp_ctx* ctx, const gp_usage_input* usage, const gp_reconcile_nodes* nodes,
                                  const gp_apps* stale /* exe_*, group, exe_count = max(0, Min - running);
                                                          drv_* and skip_if_no_fit ignored; call order = processing order */,
                                  gp_reconcile_results* out);

/* ---- node overhead (EXT/overhead.go) ---------------------------------------------------------------------------------------
 * OverheadComputer.getOverheadByNode (overhead.go:105-153) for a list of nodes, in one call: GetOverhead and
 * GetNonSchedulableOverhead together.  The event side stays with the caller: one record slot per pod the informer added
 * (addPodRequests, :163-174: spec.nodeName set, podToResources at that event -- containers summed, then a per-dimension max
 * with each init container), removed by deletePodRequests (:176-193).  Per call, for each recorded pod on a listed node:
 *   1. listed = 0 (the pod lister has no pod of the record's namespace/name): skipped (:131-138).  Everything below reads the
 *      lister's CURRENT pod.
 *   2. PodHasReservation (EXT/resourcereservations.go:115-132): false without a spark-app-id label; true when the
 *      ResourceReservation (namespace, appID) exists and lists the pod's name in Status.Pods; else true when spark-role is
 *      "executor" and the soft store's entry for appID (keyed by appID alone, no namespace) has the pod's name as a key.
 *   3. no reservation: the requests go to overhead[node] and, unless spec.schedulerName is "spark-scheduler", to
 *      nonsched[node]; a spark-scheduler pod whose application has a ResourceReservation is one the reference logs a
 *      warning for (:140-145), counted in n_warned.
 *   4. a listed node without recorded pods gets zero; records on nodes outside the list are ignored.
 * A node's value does not depend on which other nodes are listed.  Strings never cross the boundary: the caller interns node
 * names, (namespace, spark-app-id) pairs, spark-app-ids and pod names to dense ids. */
typedef struct {
    int64_t n_pods;                  /* record slots, < 2^31; a free slot has node_id = -1 and is ignored entirely */
    int32_t n_node_ids, n_app_keys, n_app_ids, n_names;
    const int32_t* node_id;          /* [n_pods] interned spec.nodeName at the add event, -1 = free slot */
    const int64_t* req_cpu_milli;    /* [n_pods] podToResources at the add event: >= 0, < 2^61 */
    const int64_t* req_mem_bytes;
    const int64_t* req_gpu;          /* or NULL (= 0) */
    const uint8_t* listed;           /* [n_pods] the lister holds a pod of this namespace/name; or NULL (= all).  The fields
                                        below describe that pod and are ignored where listed = 0 */
    const int32_t* app_key;          /* [n_pods] interned (namespace, spark-app-id), -1 = no spark-app-id label */
    const int32_t* app_id;           /* [n_pods] interned spark-app-id, -1 exactly where app_key is -1 */
    const int32_t* name_id;          /* [n_pods] interned pod name */
    const uint8_t* is_executor;      /* [n_pods] spark-role == "executor"; or NULL (= none) */
    const uint8_t* spark_scheduler;  /* [n_pods] spec.schedulerName == "spark-scheduler"; or NULL (= none) */
} gp_overhead_pods;
typedef struct {
    int32_t n_rr;                    /* ResourceReservations: distinct rr_app_key, each with its Status.Pods values */
    int32_t n_soft;                  /* soft-store entries: distinct soft_app_id, each with its Reservations keys */
    const int32_t* rr_app_key;       /* [n_rr] */
    const int64_t* rr_pod_off;       /* [n_rr + 1] CSR, starts at 0, non-decreasing */
    const int32_t* rr_pod_name;      /* name ids */
    const int32_t* soft_app_id;      /* [n_soft] */
    const int64_t* soft_pod_off;     /* [n_soft + 1] */
    const int32_t* soft_pod_name;
} gp_overhead_reservations;
typedef struct {
    int64_t* overhead_cpu_milli;     /* [n_nodes] GetOverhead, or NULL */
    int64_t* overhead_mem_bytes;
    int64_t* overhead_gpu;
    int64_t* nonsched_cpu_milli;     /* [n_nodes] GetNonSchedulableOverhead, or NULL */
    int64_t* nonsched_mem_bytes;
    int64_t* nonsched_gpu;
    uint8_t* has_reservation;        /* [n_pods] PodHasReservation of every listed record (0 for free and unlisted slots), or NULL */
    int64_t* n_warned;               /* pods on listed nodes counted by step 3's warning, or NULL */
} gp_overhead_out;
/* The outputs are in the order of node_ids (the caller's node table) and can be passed unchanged as gp_usage_input.overhead_*
 * or gp_capacity_nodes.overhead_*.  The context is left alone (snapshot, SchedulableResources, zone layout, held az-aware
 * orders, gp_last_stats); scratch of its own, one stream synchronise.
 * GP_ERR_INVALID (gp_last_error names the cause): missing arrays or negative sizes; a node, app-key, app-id or name id out of
 * range; app_key and app_id disagreeing on -1; a node id listed twice in node_ids, or an rr_app_key / soft_app_id given twice;
 * CSR offsets that do not start at 0 or decrease; a negative request.  GP_ERR_UNREPRESENTABLE: a request >= 2^61 or a
 * per-node sum >= 2^61 (the whole call is refused, nothing wraps).  On an error the outputs are undefined. */
gp_status gp_node_overhead(gp_ctx* ctx, const gp_overhead_pods* pods, const gp_overhead_reservations* rsv, int32_t n_nodes,
                           const int32_t* node_ids /* [n_nodes] the listed nodes, in node-table order */, gp_overhead_out* out);

/* ---- the resident overhead table ------------------------------------------------------------------------------------------
 * The same computation as gp_node_overhead over state the context keeps on the device and changes only by deltas, so a
 * Predicate uploads the listed node ids alone instead of every record and reservation entry.  The state:
 *   record slots   [n_slots] rows with the columns of gp_overhead_pods; node_id = -1 marks a free slot
 *   RR flags       one per app key: the ResourceReservation (namespace, spark-app-id) exists
 *   member set     (kind, app, name) triples: kind 0 = (app key, pod name) for a name in a ResourceReservation's Status.Pods,
 *                  kind 1 = (app id, pod name) for a key in the soft store entry of that app id
 * A query answers exactly what gp_node_overhead answers for: the slots as gp_overhead_pods, rr_app_key = the app keys whose RR
 * flag is set, each listing its kind-0 members, soft_app_id = the app ids that have kind-1 members.  Kind-0 members of an app
 * key whose flag is clear are never read; as in gp_node_overhead, free slots are ignored and the pod fields of a slot with
 * listed = 0 are not read.  The table belongs to the context (freed by gp_destroy); no other entry reads or changes it. */
typedef struct {
    int64_t n_slots;                                        /* slot capacity, < 2^31 */
    int32_t n_node_ids, n_app_keys, n_app_ids, n_names;     /* id capacities */
} gp_overhead_table_size;
/* Replace the context's table with an empty one of these capacities: every slot free, no RR flag, no member.
 * GP_ERR_INVALID: NULL size, a negative capacity or n_slots >= 2^31 (the table held before is kept).  After a CUDA error
 * the context holds no table. */
gp_status gp_overhead_table_reset(gp_ctx* ctx, const gp_overhead_table_size* size);

typedef struct {
    int64_t n_write;                 /* slot writes: each the slot's whole new row; node_id = -1 frees the slot */
    const int32_t* slot;             /* [n_write] distinct, < n_slots */
    const int32_t* node_id;          /* [n_write] the columns of gp_overhead_pods, with its NULL conventions: */
    const int64_t* req_cpu_milli;    /*   req_gpu NULL = 0, listed NULL = all, is_executor and spark_scheduler NULL = none */
    const int64_t* req_mem_bytes;
    const int64_t* req_gpu;
    const uint8_t* listed;
    const int32_t* app_key;
    const int32_t* app_id;
    const int32_t* name_id;
    const uint8_t* is_executor;
    const uint8_t* spark_scheduler;
    int32_t n_rr;                    /* RR flag writes */
    const int32_t* rr_app_key;       /* [n_rr] distinct */
    const uint8_t* rr_exists;        /* [n_rr] nonzero = the flag is set */
    int64_t n_member;                /* member writes: present nonzero inserts (a present triple: no-op), 0 removes (an absent
                                        one: no-op) */
    const uint8_t* member_kind;      /* [n_member] 0 = RR (member_app is an app key), 1 = soft (member_app is an app id) */
    const int32_t* member_app;
    const int32_t* member_name;
    const uint8_t* member_present;   /* the triples (kind, app, name) are distinct */
} gp_overhead_delta;
/* Apply one delta.  The whole delta is checked on the device before anything is written: a refused delta leaves the table
 * exactly as it was.  The order in which the writes of one delta apply is not observable.  One stream synchronise.
 * GP_ERR_INVALID: no table (gp_overhead_table_reset first), missing arrays or negative counts; a slot or id outside its
 * capacity or a member kind other than 0 and 1; a slot, rr_app_key or member triple given twice; app_key and app_id disagreeing
 * on -1 (listed rows); a negative request (rows with node_id != -1).  GP_ERR_UNREPRESENTABLE: a request >= 2^61, so no table
 * ever holds one.  GP_ERR_CAPACITY: more than 2^29 members.  A refusal, or a CUDA error while the delta is staged, leaves the
 * table as it was; a CUDA error once the update writes the table's buffers leaves no table (GP_ERR_INVALID "no overhead
 * table" until the next reset), and the caller resets and replays its whole state. */
gp_status gp_overhead_table_update(gp_ctx* ctx, const gp_overhead_delta* delta);
/* GetOverhead and GetNonSchedulableOverhead of the listed nodes from the table: node_ids is the only upload, and only the
 * outputs asked for come back (48 bytes per listed node, has_reservation [n_slots], n_warned).  The outputs are those of
 * gp_node_overhead on the equivalent arrays.  GP_ERR_INVALID: no table, missing arrays or a negative count, a node id out of
 * range or listed twice.  GP_ERR_UNREPRESENTABLE: a per-node sum >= 2^61.  A query never changes the table. */
gp_status gp_overhead_table_query(gp_ctx* ctx, int32_t n_nodes, const int32_t* node_ids, gp_overhead_out* out);

/* ---- the resident reservation table ---------------------------------------------------------------------------------------
 * GetReservedResources' rows (every ResourceReservation's Spec.Reservations entry and every soft reservation, hard and soft
 * alike) kept on the device and changed only by deltas, so a Predicate no longer uploads one gp_usage_input row per
 * reservation.  The state: [n_slots] slots, each a reservation-table node id (-1 = free slot) and cpu / mem / gpu.  Node ids are
 * the caller's interned node names; a row whose node has left the cluster keeps its id and is ignored where no node-table
 * entry carries that id, like the map lookup at resources.go:72-75.  The table belongs to the context (freed by gp_destroy);
 * updates change no snapshot, layout, schedulable resources or statistics. */
typedef struct {
    int64_t n_slots;                 /* slot capacity, < 2^31 */
    int32_t n_node_ids;              /* node id capacity */
} gp_reservation_table_size;
/* Replace the context's reservation table with an empty one (every slot free).  GP_ERR_INVALID: NULL size, a negative
 * capacity or n_slots >= 2^31 (the table held before is kept).  After a CUDA error the context holds no table. */
gp_status gp_reservation_table_reset(gp_ctx* ctx, const gp_reservation_table_size* size);

typedef struct {
    int64_t n_write;                 /* whole-row slot writes; node_id = -1 frees the slot */
    const int32_t* slot;             /* [n_write] distinct, < n_slots */
    const int32_t* node_id;          /* [n_write] in [-1, n_node_ids) */
    const int64_t* cpu_milli;        /* [n_write] any value with |v| < 2^61 (negative included, as gp_usage_input accepts) */
    const int64_t* mem_bytes;
    const int64_t* gpu;              /* or NULL (= 0) */
} gp_reservation_delta;
/* Apply one delta.  The whole delta is checked on the device before anything is written: a refused delta leaves the table
 * exactly as it was.  One stream synchronise.  GP_ERR_INVALID: no table (gp_reservation_table_reset first), missing arrays or
 * a negative count; a slot or node id out of range; a slot given twice.  GP_ERR_UNREPRESENTABLE: |cpu|, |mem| or |gpu| >= 2^61
 * on a row with node_id != -1.  A refusal, or a CUDA error while the delta is staged, leaves the table as it was; a CUDA error
 * once the update writes the table leaves no table (GP_ERR_INVALID "no reservation table" until the next reset), and the
 * caller resets and replays its whole state. */
gp_status gp_reservation_table_update(gp_ctx* ctx, const gp_reservation_delta* delta);

/* The node table of the resident Predicate front ends: allocatable and overhead as in gp_usage_input, and the reservations
 * from the resident table.  Overhead comes either from the host arrays (NULL = 0) or, with overhead_node_id given, from the
 * resident overhead table on the device (GetOverhead, gp_overhead_table_query's overhead_*), never crossing to the host. */
typedef struct {
    int32_t n_nodes;
    const int32_t* node_id;            /* [n_nodes] reservation-table id of each node-table entry, distinct, -1 = none */
    const int64_t* alloc_cpu_milli;    /* [n_nodes] as gp_usage_input */
    const int64_t* alloc_mem_bytes;
    const int64_t* alloc_gpu;          /* or NULL (= 0) */
    const int32_t* overhead_node_id;   /* [n_nodes] overhead-table ids (distinct, -1 = no records), or NULL = overhead_* below */
    const int64_t* overhead_cpu_milli; /* as gp_usage_input (ignored when overhead_node_id is given) */
    const int64_t* overhead_mem_bytes;
    const int64_t* overhead_gpu;
} gp_resident_usage;
/* The resident forms of gp_prepare_cluster_groups, gp_prepare_cluster_zones_groups and gp_reschedule_from_reservations: the
 * same arguments with a gp_resident_usage in place of the gp_usage_input, and the same result -- outputs bit for bit, status,
 * and the context afterwards -- as the per-call entry given the equivalent gp_usage_input: the same n_nodes and allocatable;
 * as overhead the host arrays, or gp_overhead_table_query(overhead_node_id)'s GetOverhead; one row per occupied slot with
 * res_node = the index i where node_id[i] equals the slot's id, or -1 when no entry has that id.  instance_group == NULL
 * gives gp_prepare_cluster / gp_prepare_cluster_zones, as for the per-call forms.  Uploads: the two id arrays, allocatable
 * and host overhead; the slots are read where they are.  Refusals, besides the per-call entry's (a refused call replaces
 * nothing): GP_ERR_INVALID for no reservation table, overhead_node_id without a live overhead table, an id out of range or
 * given twice; GP_ERR_UNREPRESENTABLE for a per-node overhead sum >= 2^61 (gp_overhead_table_query's refusal). */
gp_status gp_prepare_cluster_groups_resident(gp_ctx* ctx, const gp_resident_usage* usage, const gp_sort_input* sort,
                                             const int32_t* instance_group, int32_t n_instance_groups, gp_instance_group_orders* out);
gp_status gp_prepare_cluster_zones_groups_resident(gp_ctx* ctx, const gp_resident_usage* usage, const gp_sort_input* sort,
                                                   const int32_t* instance_group, int32_t n_instance_groups,
                                                   gp_instance_group_layout* layout);
gp_status gp_reschedule_from_reservations_resident(gp_ctx* ctx, const gp_resident_usage* usage, const gp_sort_input* sort,
                                                   const gp_reschedule_scope* scope, const gp_reschedule* in,
                                                   int32_t* node_out, uint8_t* ambiguous);
/* The failover reconciler's resident form: gp_reconcile_find_nodes with a gp_resident_usage in place of the gp_usage_input, on
 * the same terms as the three entries above -- placed, executor_nodes, the avail_* outputs, the status and the gp_last_error
 * category are those of gp_reconcile_find_nodes given the equivalent gp_usage_input, and the context (reservation table,
 * overhead table, snapshot, zone layout, held az-aware orders, gp_last_stats) is left as it was.  Its refusals are
 * gp_reconcile_find_nodes' and the resident ones listed above; n_nodes == 0 still gives placed = -1 for every driver without
 * reading either table (a live reservation table is still required). */
gp_status gp_reconcile_find_nodes_resident(gp_ctx* ctx, const gp_resident_usage* usage, const gp_reconcile_nodes* nodes,
                                           const gp_apps* stale, gp_reconcile_results* out);
/* The unschedulable-pod marker's resident forms: gp_exceeds_cluster_capacity[_affinity] with GetNonSchedulableOverhead from the
 * resident overhead table in place of nodes->overhead_* (ignored).  overhead_node_id [n_nodes]: the overhead-table id of each
 * node-table entry, distinct, -1 = no records (overhead 0); NULL only with n_nodes == 0.  The result -- exceeds,
 * affinity_error and the status -- is that of the per-call entry given overhead_* = gp_overhead_table_query(overhead_node_id)'s
 * nonsched_* (0 where the id is -1); the overhead is summed on the device into the call's scratch and never crosses to the
 * host.  The context, the overhead table included, is left as it was.  Refusals, besides the per-call entry's: GP_ERR_INVALID
 * for no overhead table, overhead_node_id missing, an id out of range or given twice; GP_ERR_UNREPRESENTABLE for a per-node
 * sum >= 2^61 (gp_overhead_table_query's refusal). */
gp_status gp_exceeds_cluster_capacity_resident(gp_ctx* ctx, const gp_capacity_nodes* nodes /* overhead_* ignored */,
                                               const int32_t* overhead_node_id, const gp_apps* drivers, gp_binpacker packer,
                                               uint8_t* exceeds /* [n_apps] */);
gp_status gp_exceeds_cluster_capacity_affinity_resident(gp_ctx* ctx, const gp_capacity_nodes* nodes, const int32_t* overhead_node_id,
                                                        const gp_node_labels* labels, const gp_node_affinities* affinities,
                                                        const gp_apps* drivers, gp_binpacker packer, uint8_t* exceeds /* [n_apps] */,
                                                        uint8_t* affinity_error /* [n_apps] or NULL */);

/* ---- the resident label table -------------------------------------------------------------------------------------------
 * Every node's labels kept on the device and changed only by deltas, so a driver Predicate and the marker's affinity sweep no
 * longer upload every label of every node (gp_node_labels) per call.  The state:
 *   rows          [n_node_ids] fixed-stride rows: label-table node id r owns entries [r * max_labels, r * max_labels + count[r])
 *                 of two columns, key id and value id, keys strictly ascending (node.Labels is a map); count 0 = no labels
 *   value columns [n_values] val_int_ok / val_int: strconv.ParseInt(value, 10, 64) of each interned value string -- a
 *                 function of the string, so kept per value id rather than per label
 * Node, key and value ids are the caller's interned node names, label keys and label values.  A node with more labels than
 * max_labels does not fit: the caller resets with a larger stride and replays.  The table belongs to the context (freed by
 * gp_destroy); updates change no snapshot, layout, schedulable resources, held orders or statistics. */
typedef struct {
    int32_t n_node_ids;              /* rows */
    int32_t max_labels;              /* row stride; n_node_ids * max_labels < 2^31 */
    int32_t n_keys;                  /* label key ids 0..n_keys-1 */
    int32_t n_values;                /* label value ids 0..n_values-1 */
} gp_label_table_size;
/* Replace the context's label table with an empty one: every row without labels, no value parses.  GP_ERR_INVALID: NULL
 * size, a negative capacity or n_node_ids * max_labels >= 2^31 (the table held before is kept).  After a CUDA error the
 * context holds no table. */
gp_status gp_label_table_reset(gp_ctx* ctx, const gp_label_table_size* size);

typedef struct {
    int32_t n_rows;                  /* whole-row writes: the row's new labels replace all its old ones */
    int32_t n_values;                /* value writes */
    const int32_t* row_node;         /* [n_rows] distinct node ids < n_node_ids */
    const int64_t* row_off;          /* [n_rows + 1] CSR: row_node[i]'s labels are [row_off[i], row_off[i+1]); row_off[0] = 0;
                                        an empty run clears the row (a deleted node) */
    const int32_t* label_key;        /* key ids, strictly ascending within a row */
    const int32_t* label_val;        /* value ids */
    const int32_t* value_id;         /* [n_values] distinct value ids < n_values */
    const uint8_t* value_int_ok;     /* [n_values] ParseInt(value, 10, 64) succeeded */
    const int64_t* value_int;        /* [n_values] its result where value_int_ok (ignored elsewhere) */
} gp_label_delta;
/* Apply one delta.  The whole delta is checked on the device before anything is written: a refused delta leaves the table
 * exactly as it was.  One stream synchronise.  GP_ERR_INVALID: no table (gp_label_table_reset first), missing arrays, a
 * negative count or row_off that does not start at 0 or decreases; a node or value id out of range or given twice; a row
 * longer than max_labels; a key id out of range or the keys of a row not strictly ascending; a label value id out of range.
 * A refusal, or a CUDA error while the delta is staged, leaves the table as it was; a CUDA error once the update writes the
 * table leaves no table (GP_ERR_INVALID "no label table" until the next reset), and the caller resets and replays. */
gp_status gp_label_table_update(gp_ctx* ctx, const gp_label_delta* delta);

/* The node table of a resident match: for each node-table entry its label-table id, or -1 for a node without labels.  The
 * ids may repeat: the call only reads the rows. */
typedef struct {
    int32_t n_nodes;
    int32_t reserved;
    const int32_t* node_id;          /* [n_nodes] in [-1, n_node_ids); NULL only with n_nodes == 0 */
} gp_resident_labels;
/* gp_match_node_affinity over the label table: member, n_match, n_error and the status are those of gp_match_node_affinity
 * given the equivalent gp_node_labels -- n_nodes, the table's n_keys / n_values, node i's labels = row node_id[i] (none for
 * -1), label_int_ok / label_int from the value columns.  Affinity key and value ids are checked against the table's n_keys /
 * n_values, metadata.name node indices against labels->n_nodes.  Uploads: the node ids and the programs.  The context, the
 * table included, is left alone; one stream synchronise.  Refusals: gp_match_node_affinity's for the programs, and
 * GP_ERR_INVALID for no label table or a node id outside [-1, n_node_ids). */
gp_status gp_match_node_affinity_resident(gp_ctx* ctx, const gp_resident_labels* labels, const gp_node_affinities* affinities,
                                          gp_affinity_match* out);
/* gp_exceeds_cluster_capacity_affinity_resident with the labels from the label table: its result -- exceeds, affinity_error
 * and the status -- is that of gp_exceeds_cluster_capacity_affinity_resident given the equivalent gp_node_labels (as for
 * gp_match_node_affinity_resident); labels->n_nodes = nodes->n_nodes.  Both tables are read in place and left as they were.
 * Refusals: gp_exceeds_cluster_capacity_affinity_resident's and gp_match_node_affinity_resident's. */
gp_status gp_exceeds_cluster_capacity_affinity_label_table(gp_ctx* ctx, const gp_capacity_nodes* nodes, const int32_t* overhead_node_id,
                                                           const gp_resident_labels* labels, const gp_node_affinities* affinities,
                                                           const gp_apps* drivers, gp_binpacker packer, uint8_t* exceeds /* [n_apps] */,
                                                           uint8_t* affinity_error /* [n_apps] or NULL */);

/* ---- the resident node table --------------------------------------------------------------------------------------------
 * Every node's allocatable, Spec.Unschedulable, NodeReady condition and name order kept on the device and changed only by
 * deltas from node events, so a Predicate no longer uploads those columns, nor sorts the node names on the host.  One row per
 * node id; node ids are the label table's (one node informer interns both).  A row holds: present, alloc cpu / mem / gpu,
 * unschedulable, ready, name_key, creation (the failover reconciler's newest-first order), and name_rank -- the dense rank
 * of name_key among the present rows, recomputed on the device by every update.  name_key is an order key the caller keeps: strictly increasing in the byte order of the node
 * names, unique among present rows, below 2^63 - 1, and not necessarily dense (INTEGRATION.md: a new name takes the midpoint
 * of its neighbours' keys; when no gap is left every node is relabelled in one delta).  A rank over the whole table orders
 * any subset of it as the names do.  The table belongs to the context (freed by gp_destroy); updates change no snapshot,
 * layout, schedulable resources, held orders or statistics. */
typedef struct {
    int32_t n_node_ids;              /* rows */
    int32_t reserved;
} gp_node_table_size;
/* Replace the context's node table with an empty one (no row present).  GP_ERR_INVALID: NULL size or a negative capacity
 * (the table held before is kept).  After a CUDA error the context holds no table. */
gp_status gp_node_table_reset(gp_ctx* ctx, const gp_node_table_size* size);

typedef struct {
    int32_t n_write;                 /* whole-row writes */
    int32_t reserved;
    const int32_t* node_id;          /* [n_write] distinct node ids < n_node_ids */
    const uint8_t* present;          /* [n_write] 0: the node is deleted (the row's other columns are ignored) */
    const int64_t* alloc_cpu_milli;  /* [n_write] |v| < 2^61 on present rows */
    const int64_t* alloc_mem_bytes;
    const int64_t* alloc_gpu;        /* or NULL (= 0) */
    const uint8_t* unschedulable;    /* [n_write] node.Spec.Unschedulable */
    const uint8_t* ready;            /* [n_write] NodeReady == True */
    const int64_t* name_key;         /* [n_write] the name's order key (see above) */
    const int64_t* creation;         /* [n_write] metav1.Time as UnixNano (the order of gp_reconcile_nodes.creation), or NULL
                                        (= 0 for every written row); no part of name_rank, no refusal */
} gp_node_delta;
/* Apply one delta, then recompute name_rank.  The whole delta is checked on the device before anything is written: a refused
 * delta leaves the table exactly as it was.  One stream synchronise.  GP_ERR_INVALID: no table (gp_node_table_reset first),
 * missing arrays or a negative count; a node id out of range or given twice; two rows present after the delta with the same
 * name_key, or a present row's name_key = 2^63 - 1.  GP_ERR_UNREPRESENTABLE: |alloc| >= 2^61 on a present row.  A refusal,
 * or a CUDA error while the delta is staged, leaves the table as it was; a CUDA error once the update writes the table
 * leaves no table (GP_ERR_INVALID "no node table" until the next reset), and the caller resets and replays. */
gp_status gp_node_table_update(gp_ctx* ctx, const gp_node_delta* delta);

/* The node list of a node-table Predicate entry.  Per listed node i: its node-table id, its reservation-table id and its
 * overhead-table id -- the only per-node uploads, with is_driver_candidate when given.  Per call: how the zone, the instance
 * group and the two label priority ranks are read from the label table's row node_table_id[i] (the reference's rules):
 *   zone            label zone_key (failure-domain.beta.kubernetes.io/zone); the dense zone is the index of its value id in
 *                   zone_value [n_zones]; a node without the label is in zone zone_missing (the "default" placeholder's
 *                   dense id), or is refused when zone_missing = -1; a value not listed is refused.  zone_key = -1: one
 *                   zone (zone_id NULL of gp_sort_input).
 *   instance group  label instance_group_key; the index of its value id in instance_group_value [n_instance_groups of the
 *                   entry]; a node without the label or with a value not listed is in no instance group (-1).  Ignored when
 *                   the entry is given an instance_group array; key -1 without one: every node in instance group 0.
 *   label ranks     label driver_rank_key / executor_rank_key; the rank is the index of the value id in the list
 *                   (DescendingPriorityValues order, the last index of a repeated value); -1 without the label or for a
 *                   value not listed (extractRank's false).  Key -1: not configured (the gp_sort_input column NULL). */
typedef struct {
    int32_t n_nodes;
    int32_t reserved;
    const int32_t* node_table_id;        /* [n_nodes] distinct, each a present row */
    const int32_t* reservation_id;       /* [n_nodes] as gp_resident_usage.node_id (NULL for the marker's entries) */
    const int32_t* overhead_node_id;     /* [n_nodes] as gp_resident_usage.overhead_node_id; required */
    const uint8_t* is_driver_candidate;  /* [n_nodes] member of ExtenderArgs.NodeNames, or NULL (= all) */
    int32_t zone_key;
    int32_t n_zones;                     /* >= 1 */
    const int32_t* zone_value;           /* [n_zones] distinct value ids, or NULL with zone_key = -1 */
    int32_t zone_missing;                /* in [-1, n_zones) */
    int32_t instance_group_key;
    const int32_t* instance_group_value; /* [n_instance_groups] distinct value ids, or NULL with instance_group_key = -1 */
    int32_t driver_rank_key;
    int32_t n_driver_rank_values;
    const int32_t* driver_rank_value;
    int32_t executor_rank_key;
    int32_t n_executor_rank_values;
    const int32_t* executor_rank_value;
    int32_t* undefined_ties;             /* out, or NULL: as gp_sort_input.undefined_ties */
    int32_t* zone_id_out;                /* out [n_nodes], or NULL: the dense zone of each node (0 with zone_key = -1) */
    int32_t* instance_group_out;         /* out [n_nodes], or NULL: the instance group of each node */
} gp_node_table_nodes;
/* The node-table forms of the three *_resident Predicate entries: a gp_node_table_nodes in place of both the
 * gp_resident_usage and the gp_sort_input.  One kernel gathers, on the device, exactly the columns the *_resident entry would
 * upload (allocatable, name_rank, unschedulable and ready from the node table; zone, instance group and label ranks from the
 * label table), and the *_resident entry's stages then run unchanged.  So each returns what its *_resident entry returns --
 * outputs bit for bit, status, and the context afterwards -- given node_id = reservation_id, overhead from the overhead
 * table, and the columns above.  The node and label tables are read in place and left as they were.
 * Checks, in order (a refused call replaces nothing): GP_ERR_INVALID for no node table, no label table, missing arrays
 * (overhead_node_id included) or bad sizes, a zone_missing out of range, a value listed twice in zone_value or
 * instance_group_value; then the *_resident entry's host checks; then, read in the one synchronise the entry makes before it
 * writes the context, GP_ERR_INVALID for a node-table id out of range, absent or given twice, and for a zone label whose
 * value is not in zone_value (or a node without it when zone_missing = -1); then the *_resident entry's device refusals. */
gp_status gp_prepare_cluster_groups_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, const int32_t* instance_group,
                                               int32_t n_instance_groups, gp_instance_group_orders* out);
gp_status gp_prepare_cluster_zones_groups_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, const int32_t* instance_group,
                                                     int32_t n_instance_groups, gp_instance_group_layout* layout);
gp_status gp_reschedule_from_reservations_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, const gp_reschedule_scope* scope,
                                                     const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous);
/* The failover reconciler's node-table form: gp_reconcile_find_nodes_resident with the node columns gathered on the device.
 * It returns what gp_reconcile_find_nodes_resident returns -- placed, executor_nodes, the avail_* outputs, the status and
 * the gp_last_error category -- and leaves the context as it does, given node_id = reservation_id, allocatable from the
 * node table, overhead from the overhead table, and gp_reconcile_nodes{n_groups, node_group = the groups below, creation,
 * unschedulable and ready from the node table}.  is_driver_candidate and the rank keys are ignored.
 * The instance group follows the reference's instanceGroup(n.Labels[instanceGroupLabel]), where a missing label reads "":
 *   instance_group_key >= 0   the index of the node's value id in instance_group_value [n_groups]; a node without the label
 *                             is in instance_group_missing, the dense id of "" (list the value id of "" there, or -1 when no
 *                             node carries ""), and is refused when instance_group_missing = -1; a value not listed is
 *                             refused (every node must lie in [0, n_groups)).
 *   instance_group_key = -1   every node in group 0.
 * instance_group_out, when given, receives these groups.  Checks, in order (a refused call changes no state; its outputs
 * are undefined): the gather's host checks (as for the entries above, and instance_group_missing outside [-1, n_groups)); then
 * gp_reconcile_find_nodes_resident's host checks; then, read in its one synchronise, a node-table id out of range, absent
 * or given twice, a zone refusal (zone_key >= 0), and an instance-group refusal; then its device refusals.  Like the
 * resident form, a call with n_nodes = 0, or without stale drivers and avail_* outputs, returns before any device work is
 * read. */
gp_status gp_reconcile_find_nodes_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, int32_t n_groups,
                                             int32_t instance_group_missing, const gp_apps* stale, gp_reconcile_results* out);
/* The unschedulable-pod marker's node-table forms: gp_exceeds_cluster_capacity_resident and
 * gp_exceeds_cluster_capacity_affinity_label_table with allocatable gathered from the node table, zone_id from the label
 * table (zone_key, zone_value, zone_missing as above; NULL with zone_key = -1), overhead_node_id from nodes, and (affinity
 * form) the label rows node_table_id.  Each returns what that entry returns -- exceeds, affinity_error and the status --
 * and leaves the context as it does.  Unschedulable and not-ready nodes count, as in the marker.  reservation_id may be NULL;
 * is_driver_candidate, the instance-group and rank keys are ignored.  node_group / n_groups: as gp_capacity_nodes'.
 * Checks, in order: affinities missing (affinity form, as gp_exceeds_cluster_capacity_affinity_label_table checks first), the
 * gather's host checks, the entry's host checks, then in its one synchronise the gather's refusals (a node-table id out of
 * range, absent or given twice; a zone), then the entry's device refusals. */
gp_status gp_exceeds_cluster_capacity_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, const int32_t* node_group,
                                                 int32_t n_groups, const gp_apps* drivers, gp_binpacker packer,
                                                 uint8_t* exceeds /* [n_apps] */);
gp_status gp_exceeds_cluster_capacity_affinity_node_table(gp_ctx* ctx, const gp_node_table_nodes* nodes,
                                                          const gp_node_affinities* affinities, const gp_apps* drivers,
                                                          gp_binpacker packer, uint8_t* exceeds /* [n_apps] */,
                                                          uint8_t* affinity_error /* [n_apps] or NULL */);

/* ---- the resident driver table (pending drivers from the pod informer) --------------------------------------------------
 * Every pending, parseable driver pod kept on the device and changed only by deltas from pod events, so that a FIFO
 * Predicate no longer lists, sorts, parses and uploads the queue of earlier drivers (ListEarlierDrivers, EXT/sparkpods.go:54-71;
 * sparkResources and shouldSkipDriverFifo, EXT/resource.go:224-270).  One row per slot; the host interns instance-group names
 * (FindInstanceGroupFromPodSpec) and Spec.SchedulerName into dense ids.  A row holds: present, creation (CreationTimestamp as
 * UnixNano), scheduler, group (-1: no instance group found -- MatchPodInstanceGroup is then false for every pair), the six
 * quantities of sparkResources, min_executor_count (MinExecutorCount, the only count that packs) and exact (0: a quantity lies
 * outside the exact-int64 model).  The host writes only pending drivers whose annotations parse: a driver that is bound,
 * deleted, carries a DeletionTimestamp or no longer parses is cleared (EXT/resource.go:232-237 skips it).  The table belongs to
 * the context (freed by gp_destroy); updates change no snapshot, layout, schedulable resources, held orders or statistics. */
typedef struct {
    int32_t n_slots;                 /* rows */
    int32_t n_groups;                /* instance-group ids 0 .. n_groups-1 */
    int32_t n_schedulers;            /* scheduler ids 0 .. n_schedulers-1 */
    int32_t reserved;
} gp_driver_table_size;
/* Replace the context's driver table with an empty one (no row present).  GP_ERR_INVALID: NULL size or a negative capacity
 * (the table held before is kept).  After a CUDA error the context holds no table. */
gp_status gp_driver_table_reset(gp_ctx* ctx, const gp_driver_table_size* size);

typedef struct {
    int32_t n_write;                 /* whole-slot writes */
    int32_t reserved;
    const int32_t* slot;             /* [n_write] distinct slots < n_slots */
    const uint8_t* present;          /* [n_write] 0: the slot is cleared (the other columns are ignored) */
    const int64_t* creation;         /* [n_write] CreationTimestamp as UnixNano */
    const int32_t* scheduler;        /* [n_write] in [0, n_schedulers) on present rows */
    const int32_t* group;            /* [n_write] in [-1, n_groups) on present rows */
    const int64_t* drv_cpu_milli;    /* [n_write] as gp_apps' columns; negative values are kept (the pack refuses them) */
    const int64_t* drv_mem_bytes;
    const int64_t* drv_gpu;          /* or NULL (= 0) */
    const int64_t* exe_cpu_milli;
    const int64_t* exe_mem_bytes;
    const int64_t* exe_gpu;          /* or NULL (= 0) */
    const int32_t* min_executor_count;
    const uint8_t* exact;            /* [n_write] 0: a quantity is outside the exact-int64 model (the row queues, but a queue that
                                        selects it is refused with GP_ERR_UNREPRESENTABLE) */
    const int32_t* affinity;         /* [n_write] the driver's required-affinity id in the caller's affinity interner; -1: no
                                        nodeSelector and no required node affinity (matches every node).  NULL writes -1.  Not
                                        checked here: its range is the sweep's gp_node_affinities, checked by
                                        gp_exceeds_cluster_capacity_driver_table.  The FIFO entries do not read it. */
} gp_driver_delta;
/* Apply one delta.  The whole delta is checked on the device before anything is written: a refused delta leaves the table
 * exactly as it was.  One stream synchronise.  GP_ERR_INVALID: no table (gp_driver_table_reset first), missing arrays or a
 * negative count; a slot out of range or given twice; on a present row a scheduler or group out of range.
 * GP_ERR_UNREPRESENTABLE: |quantity| >= 2^61 on a present row with exact = 1.  A refusal, or a CUDA error while the delta is
 * staged, leaves the table as it was; a CUDA error once the update writes the table leaves no table (GP_ERR_INVALID "no
 * driver table" until the next reset), and the caller resets and replays. */
gp_status gp_driver_table_update(gp_ctx* ctx, const gp_driver_delta* delta);

/* The FIFO queue one call selects from the driver table and orders on the device, and the gp_apps it packs.
 *   Predicate form (requesting_slot >= 0): selectDriverNode's ListEarlierDrivers + fitEarlierDrivers + the driver's own
 *     pack.  The queue is the present rows with the requesting row's scheduler, its group (group != -1) and a creation
 *     strictly below the requesting row's, ordered by (creation, slot); then the requesting row itself with skip_if_no_fit 0.
 *     Every entry packs in snapshot group predicate_group.  The requesting driver's driver_node is then -2
 *     (failure-earlier-driver), -1 (failure-fit) or its driver node.
 *   Drain form (requesting_slot = -1): every present row with scheduler `scheduler` and snapshot_group[row.group] >= 0, in
 *     snapshot group snapshot_group[row.group], ordered by (snapshot group, creation, slot).
 * skip_if_no_fit of a queued row = creation + enforce_after_ns[row.group] > now_unix_nano (shouldSkipDriverFifo), evaluated
 * exactly (no overflow; a negative age is allowed).  Equal creation times (whole seconds in the API) leave the reference's
 * sort.Slice order undefined: ties are broken by slot, and undefined_ties counts the adjacent entries of one queue with equal
 * creation (a shim that wants the reference's own unspecified order falls back to Go).
 * Outputs: queue_slot[i] = the slot of entry i, exec_out_off [n_queued + 1] = its ExecutorNodes offsets (the prefix sum of
 * max(min_executor_count, 0)), *n_queued and *n_executors (= exec_out_off[n_queued]).
 * Refusals, all before any pack work and changing nothing (the outputs above excepted): GP_ERR_INVALID for an absent requesting
 * slot; GP_ERR_UNREPRESENTABLE for a queued row with exact = 0; GP_ERR_CAPACITY when n_queued > queue_cap or n_executors >
 * executor_nodes_cap -- *n_queued and *n_executors then hold the sizes needed, so the caller can grow its buffers and retry. */
typedef struct {
    int32_t requesting_slot;         /* >= 0: Predicate form; -1: drain form */
    int32_t scheduler;               /* drain form: the scheduler id drained (Predicate form: ignored, the requesting row's) */
    int32_t predicate_group;         /* Predicate form: the snapshot group of every entry (normally 0) */
    int32_t queue_cap;               /* entries of queue_slot and of the results' driver_node */
    const int32_t* snapshot_group;   /* drain form: [n_groups] the snapshot group of each table group, -1 = not drained */
    const int64_t* enforce_after_ns; /* [n_groups] the FIFO age of each table group (DefaultEnforceAfterPodAge unless overridden) */
    int64_t now_unix_nano;
    int32_t* queue_slot;             /* out [queue_cap] */
    int64_t* exec_out_off;           /* out [queue_cap + 1], or NULL */
    int32_t* n_queued;               /* out */
    int64_t* n_executors;            /* out, or NULL */
    int32_t* undefined_ties;         /* out, or NULL */
} gp_driver_queue;
/* gp_pack_batch(algo GP_TIGHTLY_PACK / GP_DISTRIBUTE_EVENLY, mode GP_MODE_FIFO_REFERENCE / GP_MODE_FIFO_EXACT) on the queue,
 * over the held snapshot: driver_node [n_queued] and ExecutorNodes by exec_out_off, status, gp_last_error category, gp_last_stats
 * and the snapshot left behind are what gp_pack_batch returns on the gp_apps the host would build from the same rows.  The
 * driver table is read in place and left unchanged.  Checks: gp_pack_batch's argument checks; snapshot_group (drain form) and
 * predicate_group outside [-1, snapshot groups) resp. [0, snapshot groups) are GP_ERR_INVALID; then the refusals above.  One
 * stream synchronise after the queue stage (count, executor total and refusal word), one after the pack. */
gp_status gp_pack_fifo_driver_table(gp_ctx* ctx, const gp_driver_queue* queue, gp_algo algo, gp_mode mode, gp_results* out);
/* gp_pack_fifo_zones_groups(groups == NULL) on the queue: the snapshot groups are the instance groups of the layout
 * gp_prepare_cluster_zones_groups[_node_table] left; zone, driver_node, ExecutorNodes, avg_efficiency, status, statistics and
 * the snapshot left behind are what that entry returns on the host-built gp_apps.  Checks as gp_pack_fifo_zones_groups', with
 * the snapshot-group ranges of gp_pack_fifo_driver_table, then the queue refusals. */
gp_status gp_pack_fifo_zones_groups_driver_table(gp_ctx* ctx, const gp_driver_queue* queue, gp_binpacker packer, gp_mode mode,
                                                 const gp_instance_groups* groups /* must be NULL */, gp_zone_results* out);

/* The unschedulable-pod marker's whole sweep (scanForUnschedulablePods, EXT/unschedulablepods.go:93-166) from the driver
 * table, the node table and the label table, in one call.
 *   Stale rows: present, scheduler == `scheduler` and creation + timeout_ns < now_unix_nano (CreationTimestamp.Add(timeout)
 *     .Before(now): strict), evaluated exactly in 128 bits.  Pending, not terminating and parseable hold by construction (the
 *     host clears every other driver).  They are listed in (creation, slot) order: stale_slot[i] = the slot of entry i.
 *   outcome[i] = 2 (outside the model): the row has exact = 0, a negative quantity or a negative min_executor_count -- what
 *     gp_exceeds_cluster_capacity* would refuse for the whole call.  The caller answers it with DoesPodExceedClusterCapacity
 *     on the host; exceeds[i] is 0.
 *   Otherwise exceeds[i] and outcome[i] = 1 (the driver's affinity errors on some node: ListWithPredicate fails) or 0 are,
 *     bit for bit, exceeds and affinity_error of gp_exceeds_cluster_capacity_affinity_node_table(nodes, affinities + one
 *     appended program that matches every node, drivers) on the gp_apps built from the same rows: the six quantities,
 *     exe_count = min_executor_count and group = the row's affinity id, -1 becoming the appended program.
 * Refusals, in this order, each changing no state (the outputs excepted):
 *   1. the host checks of gp_exceeds_cluster_capacity_affinity_node_table; NULL sweep or outputs, cap < 0 (GP_ERR_INVALID);
 *      no driver table (gp_driver_table_reset first);
 *   2. read in one stream synchronise after the selection: a stale row whose affinity id lies outside [-1, n_aff)
 *      (GP_ERR_INVALID); then n_stale > cap (GP_ERR_CAPACITY, *n_stale holds the size needed: grow and retry);
 *   3. the device refusals of gp_exceeds_cluster_capacity_affinity_node_table (node gather, overhead, labels, nodes).
 * The driver, node and label tables are read in place and left unchanged.  Two stream synchronises. */
typedef struct {
    int32_t scheduler;               /* table id of the scheduler swept (spark-scheduler); -1: none (selects nothing) */
    int32_t cap;                     /* entries of the outputs below */
    int64_t timeout_ns;              /* unschedulablePodTimeoutDuration, used as given */
    int64_t now_unix_nano;
    int32_t* stale_slot;             /* out [cap] the stale drivers' slots in (creation, slot) order */
    uint8_t* exceeds;                /* out [cap] !HasCapacity, where outcome = 0 */
    uint8_t* outcome;                /* out [cap] 0 answered, 1 affinity error, 2 outside the model */
    int32_t* n_stale;                /* out */
} gp_stale_sweep;
gp_status gp_exceeds_cluster_capacity_driver_table(gp_ctx* ctx, const gp_node_table_nodes* nodes, const gp_node_affinities* affinities,
                                                   const gp_stale_sweep* sweep, gp_binpacker packer);

/* ---- several GPUs of one box behind ONE host process (SURVEY 8e) -----------------------------------------------
 * The reference is a single process with a serial Predicate (internal/extender/resource.go:194-205); this handle lets
 * that process use every GPU: one gp_ctx + one worker thread per entry of `devices` (an ordinal may repeat).
 *   gp_multi_set_snapshot   every device receives the full snapshot by a direct H2D copy over its own PCIe link.
 *   gp_multi_pack_batch     GP_MODE_INDEPENDENT: the queue is cut into one contiguous block per device and every device
 *                           copies ITS placements straight into the caller's result buffers (no gather through one GPU,
 *                           no collective: the path has no exchange step).  FIFO modes: whole instance groups per device
 *                           (queues of different groups are independent: internal/extender/sparkpods.go:61,
 *                           resource.go:292-295; longest-processing-time first on applications x nodes), results are
 *                           scattered back into queue order; exec_out_off is mandatory and node_bits must be 32 there.
 *                           Results are bit-identical to gp_pack_batch_wire on one context.
 *   gp_multi_get_snapshot   after a FIFO batch: every node from the device that owned its instance group.
 *   gp_multi_group_owner    which device ran each instance group's queue in the last FIFO batch. */
typedef struct gp_multi gp_multi;
gp_status gp_multi_create(gp_multi** out, const int32_t* devices /* NULL = 0..n-1 */, int32_t n_devices);
void gp_multi_destroy(gp_multi* m);
const char* gp_multi_last_error(const gp_multi* m);
int32_t gp_multi_size(const gp_multi* m);
gp_ctx* gp_multi_ctx(gp_multi* m, int32_t i);      /* the i-th context, e.g. for gp_alloc_pinned / gp_last_stats */
gp_status gp_multi_set_snapshot(gp_multi* m, const gp_nodes* nodes);
gp_status gp_multi_pack_batch(gp_multi* m, const gp_apps_wire* apps, gp_algo algo, gp_mode mode, gp_results_wire* out);
gp_status gp_multi_get_snapshot(gp_multi* m, int64_t* avail_cpu_milli, int64_t* avail_mem_bytes, int64_t* avail_gpu);
gp_status gp_multi_group_owner(gp_multi* m, int32_t* owner /* [n_groups] */);

/* Statistics of the last gp_pack_batch* on this context (host call, synchronises the stream):
 * nodes_scanned = executor-order entries visited, drivers_tried = driver-order entries visited,
 * summed over apps -- the N_e / N_d of the algorithmic-bytes formula (DESIGN.md); gp_pack_fifo_az_aware and
 * gp_pack_batch_az_aware include the scans of their undivided fallback in both. */
typedef struct {
    int64_t nodes_scanned;
    int64_t drivers_tried;
    int64_t kernel_launches;   /* launches of this library's kernels in that call */
    int64_t pack_kernel_ns;    /* device time of the pack kernels (CUDA events on the launch stream; independent tightly/evenly:
                                  the one classify + capacity tables + decide launch and the scan of the listed applications) */
    int64_t prep_kernel_ns;    /* device time of the work before them (preparation kernel; independent tightly/evenly: 0, the
                                  one launch prepares the applications itself and nothing runs before it) */
    int64_t scan_path_apps;    /* independent tightly/evenly: applications decided by the node-order scan instead of the
                                  per-shape capacity tables (all of them with GANGPACK_TABLES=0).
                                  FIFO modes: applications decided by the whole CTA instead of warp 0 alone (every
                                  evaluated one with GANGPACK_FIFO_WARP=0).
                                  gp_pack_fifo_az_aware / gp_pack_batch_az_aware: applications for which the undivided
                                  fallback ran, placed or not */
    int64_t scan_path_nodes;   /* executor-order entries those scans visited (nodes_scanned also counts table probes) */
    int64_t reserved[1];
} gp_stats;
gp_status gp_last_stats(gp_ctx* ctx, gp_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* GANGPACK_H */
