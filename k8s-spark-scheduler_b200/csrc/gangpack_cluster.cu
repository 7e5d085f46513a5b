// gangpack_cluster.cu -- the entry points driven by the reservations: node priority orders (gp_potential_nodes),
// availability (gp_build_*availability), the prepared snapshots (gp_prepare_cluster[_groups], gp_prepare_cluster_zones[_groups]), executor
// reschedule (gp_reschedule_executors, gp_reschedule_from_reservations) and the failover reconciler (gp_reconcile_find_nodes),
// with the input checks and device staging they share; the *_resident forms of gp_prepare_cluster_groups,
// gp_prepare_cluster_zones_groups, gp_reschedule_from_reservations and gp_reconcile_find_nodes, which take the reservations
// from the resident table; and the *_node_table forms of the first three, which take the node columns from the resident node
// and label tables as well.
#include "gangpack_ctx.cuh"
#include "gangpack_sort.cuh"
#include "gangpack_zonelayout.cuh"
#include "gangpack_resched.cuh"
#include "gangpack_reschedprep.cuh"
#include "gangpack_reconcile.cuh"

#include <algorithm>
#include <string>
#include <vector>

// ---- node priority order (f1) and availability snapshot (f2): device stages + the entries built on them ----

// exec_off / drv_off [n_ig + 1] of the plain multi-group snapshot: instance group g's range of the instance-group-major
// candidate orders (ig NULL: every node in instance group 0, so [0, count, count, ...])
__global__ void gp_ig_offsets(int32_t n_ig, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv,
                              const int32_t* __restrict__ exe, const int32_t* __restrict__ ig, int32_t* __restrict__ exec_off,
                              int32_t* __restrict__ drv_off) {
    const int32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_ig) return;
    drv_off[g] = ig_lower_bound(drv, counts[0], ig, g);
    exec_off[g] = ig_lower_bound(exe, counts[1], ig, g);
}

// Host checks shared by the entries below; `who` (the entry's name) prefixes every message.  The shape of a gp_usage_input:
// sizes non-negative, the allocatable columns for nodes, the reservation columns for rows, fewer than 2^31 rows (the bound
// the exact usage sums rest on).  The quantities themselves are checked where they are read, on the device (usage_refusal).
static gp_status check_usage(gp_ctx* c, const gp_usage_input* in, const char* who) {
    if (!in || in->n_nodes < 0 || in->n_reservations < 0 || in->n_reservations > 0x7fffffffLL ||
        (in->n_nodes > 0 && (!in->alloc_cpu_milli || !in->alloc_mem_bytes)) ||
        (in->n_reservations > 0 && (!in->res_node || !in->res_cpu_milli || !in->res_mem_bytes)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes");
    return GP_OK;
}

// The status word of the availability stage (kFeErr* bits), read back by the entry: the refusal it stands for.
static const Refusal kFeRefusals[] = {
    {kFeErrId, GP_ERR_INVALID, "a reservation-table or overhead-table node id out of range or given twice"},
    {kFeErrInput, GP_ERR_UNREPRESENTABLE, "|allocatable|, |overhead| or |reservation| >= 2^61"},
    {kFeErrResult, GP_ERR_UNREPRESENTABLE, "a node's reservation sum or availability lies outside the exact-int64 domain (|v| >= 2^61)"},
};

// Where an availability stage takes its usage from: the per-call rows of a gp_usage_input, or the resident reservation table
// through a gp_resident_usage (the *_resident entries).  Everything else of the stage is the same for both.
// The *_node_table entries pass a gp_resident_usage and a gp_sort_input whose node columns were gathered on the device
// (nt_gather): gather_err, the gather's status word, marks them.
struct UsageIn {
    const gp_usage_input* rows = nullptr;
    const gp_resident_usage* res = nullptr;
    const int* gather_err = nullptr;
    UsageIn(const gp_usage_input* u) : rows(u) {}
    UsageIn(const gp_resident_usage* r, const int* gathered = nullptr) : res(r), gather_err(gathered) {}
    bool given() const { return rows || res; }
    // allocatable and the gp_sort_input columns other than is_driver_candidate are device pointers.  They are not checked on
    // the host: the gather keeps every index in range and name_rank unique even for a call it refuses, and its status word is
    // read in the entry's synchronise, before the context is written
    bool on_device() const { return gather_err != nullptr; }
    int32_t n_nodes() const { return rows ? rows->n_nodes : res ? res->n_nodes : 0; }
    // overhead from the resident overhead table, on the device
    bool table_overhead() const { return res && res->overhead_node_id; }
};

// check_usage for either source.  The resident form: the node table's columns, a live reservation table, and a live overhead
// table when overhead_node_id is given; the ids themselves are checked on the device (kFeErrId).
static gp_status check_source(gp_ctx* c, const UsageIn& u, const char* who) {
    if (!u.res) return check_usage(c, u.rows, who);
    const gp_resident_usage* r = u.res;
    if (r->n_nodes < 0 || (r->n_nodes > 0 && (!r->node_id || !r->alloc_cpu_milli || !r->alloc_mem_bytes)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes");
    GP_TRY(require(c, c->rt.need(), who));
    if (r->overhead_node_id && !c->oht.live) return fail(c, GP_ERR_INVALID, who, "overhead_node_id without an overhead table");
    return GP_OK;
}

// The two status words of the availability stage once the stream has been synchronised: err[0] kFeErr* bits, err[1] the
// overhead query's bits (resident overhead only).  Ids first, then the overhead sums, then the domain of the stage itself.
static gp_status stage_refusal(gp_ctx* c, const int* err, const char* who) {
    GP_TRY(refuse(c, err[0] & kFeErrId, kFeRefusals, who));
    GP_TRY(oht_sum_refusal(c, err[1], who));
    return refuse(c, err[0], kFeRefusals, who);
}

void enqueue_resident_dir(cudaStream_t st, int32_t n, const int32_t* ids, int32_t lim, int32_t* dir, int* d_err) {
    const int T = 256;
    if (n > 0) gp_resident_dirs<<<(n + T - 1) / T, T, 0, st>>>(n, ids, lim, dir, nullptr, 0, nullptr, d_err);
}

// The failover loop's status word (kRcErr* bits)
static const Refusal kRcRefusals[] = {
    {kRcErrDomain, GP_ERR_UNREPRESENTABLE, "an availability the loop charged lies outside the exact-int64 domain (|v| >= 2^61)"},
};

// The two id arrays of a gp_sort_input the kernels index with: zone ids in range, name ranks a permutation of 0..n-1 (a rank
// given twice would leave a position of the order unwritten).
static gp_status check_sort_ids(gp_ctx* c, const gp_sort_input* in, const char* who) {
    const int32_t n = in->n_nodes;
    if (in->zone_id) for (int32_t i = 0; i < n; ++i)
        if (in->zone_id[i] < 0 || in->zone_id[i] >= in->n_zones) return fail(c, GP_ERR_INVALID, who, "zone_id out of range");
    if (in->name_rank) {
        std::vector<uint8_t>& seen = c->v_seen_e;       // host scratch of the order checks
        seen.assign((size_t)n, 0);
        for (int32_t i = 0; i < n; ++i) {
            const int32_t r = in->name_rank[i];
            if (r < 0 || r >= n) return fail(c, GP_ERR_INVALID, who, "name_rank out of range");
            if (seen[r]) return fail(c, GP_ERR_INVALID, who, "name_rank is not a permutation (a rank is given twice)");
            seen[r] = 1;
        }
    }
    return GP_OK;
}

// Executor requests (gpu optional): non-negative and inside the exact-int64 domain.
static gp_status check_requests(gp_ctx* c, int32_t q, const int64_t* cpu, const int64_t* mem, const int64_t* gpu, const char* who) {
    for (int32_t i = 0; i < q; ++i) {
        const int64_t v[3] = {cpu[i], mem[i], gpu ? gpu[i] : 0};
        for (int64_t x : v) {
            if (x < 0) return fail(c, GP_ERR_INVALID, who, "negative resource request");
            if (x >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, who, "quantity >= 2^61");
        }
    }
    return GP_OK;
}

// The host_off / host_nodes CSR of a gp_reschedule (host_off given): monotone from 0, node indices below n_nodes.
// *hosted = host_off[n_execs].
static gp_status check_hosting(gp_ctx* c, const gp_reschedule* in, int32_t n_nodes, int64_t* hosted, const char* who) {
    if (in->host_off[0] != 0) return fail(c, GP_ERR_INVALID, who, "host_off must start at 0");
    for (int32_t i = 0; i < in->n_execs; ++i)
        if (in->host_off[i + 1] < in->host_off[i]) return fail(c, GP_ERR_INVALID, who, "host_off not monotone");
    *hosted = in->host_off[in->n_execs];
    if (*hosted > 0 && !in->host_nodes) return fail(c, GP_ERR_INVALID, who, "host_nodes missing");
    for (int64_t t = 0; t < *hosted; ++t)
        if (in->host_nodes[t] < 0 || in->host_nodes[t] >= n_nodes) return fail(c, GP_ERR_INVALID, who, "host_nodes index out of range");
    return GP_OK;
}

// f2 stage: uploads the inputs, leaves avail[3][N] / sched[3][N] and the stage's two status words (*d_err: [2], for
// stage_refusal once the stream has been synchronised) on the device (usagebuf).
// d_over (optional, [3]): the device overhead columns, NULL where the caller gave none.
// The usage sums come from the per-call rows (gp_usage_scatter<UsageRowIndex>) or from the reservation table's slots through a
// directory built from node_id (gp_resident_dirs, gp_usage_scatter<UsageSlotDir>); resident overhead is the overhead table's
// GetOverhead written straight into the overhead piece (oht_enqueue_sums).  From the sums on, both are the same kernels.
static gp_status stage_availability(gp_ctx* c, const UsageIn& in, cudaStream_t st, long long** d_avail, long long** d_sched, int** d_err,
                                    long long** d_resched = nullptr, const long long** d_over = nullptr) {
    const int32_t n = in.n_nodes();
    const gp_usage_input* rows = in.rows;
    const gp_resident_usage* res = in.res;
    const bool tab = in.table_overhead();
    const size_t N = (size_t)n, R = rows ? (size_t)rows->n_reservations : 0;
    const size_t S = res ? (size_t)c->rt.size.n_slots : 0;
    const size_t RI = res ? (size_t)c->rt.size.n_node_ids : 0, OI = tab ? (size_t)c->oht.size.n_node_ids : 0;
    const int64_t* const alloc_h[3] = {rows ? rows->alloc_cpu_milli : res->alloc_cpu_milli, rows ? rows->alloc_mem_bytes : res->alloc_mem_bytes,
                                       rows ? rows->alloc_gpu : res->alloc_gpu};
    const int64_t* const over_h[3] = {rows ? rows->overhead_cpu_milli : res->overhead_cpu_milli,
                                      rows ? rows->overhead_mem_bytes : res->overhead_mem_bytes,
                                      rows ? rows->overhead_gpu : res->overhead_gpu};
    Arena ar{c->usagebuf, st};
    // resident overhead: the query's six columns, GetOverhead first
    const auto alloc = ar.take<long long>(3 * N), over = ar.take<long long>((tab ? 6 : 3) * N);
    const auto usage = ar.take<unsigned long long>(6 * N);
    const auto has = ar.take<unsigned int>(N);
    const auto err = ar.take<int>(2);
    const auto avail = ar.take<long long>(3 * N), sched = ar.take<long long>(3 * N), resched = ar.take<long long>(3 * N);
    const auto rn = ar.take<int32_t>(R);
    const auto rc = ar.take<long long>(R), rm = ar.take<long long>(R), rg = ar.take<long long>(R);
    const auto ids = ar.take<int32_t>(res ? N : 0), oids = ar.take<int32_t>(tab ? N : 0);
    const auto rdir = ar.take<int32_t>(RI), odir = ar.take<int32_t>(OI);
    const auto acc = ar.take<unsigned long long>(tab ? 12 * N : 0), warned = ar.take<unsigned long long>(tab ? 1 : 0);
    ar.reserve();
    const long long* al[3];
    const long long* ov[3];
    for (int d = 0; d < 3; ++d) {
        al[d] = in.on_device() ? (const long long*)alloc_h[d] : ar.put(alloc.part(N * d, N), alloc_h[d]);
        ov[d] = tab ? ar.ptr(over.part(N * d, N)) : ar.put(over.part(N * d, N), over_h[d]);
    }
    ar.fill(usage, err, 0);                             // the usage sums, the has-an-entry flags and the status words
    const int T = 256;
    if (rows) {
        const int32_t* r_node = ar.put(rn, rows->res_node);
        const long long* r_cpu = ar.put(rc, rows->res_cpu_milli);
        const long long* r_mem = ar.put(rm, rows->res_mem_bytes);
        const long long* r_gpu = ar.put(rg, rows->res_gpu);
        GP_TRY(ar.check(c));
        if (R)
            gp_usage_scatter<<<(unsigned)((R + T - 1) / T), T, 0, st>>>((long long)R, UsageRowIndex{r_node, n}, r_cpu, r_mem, r_gpu, n,
                                                                       ar.ptr(usage), d_resched ? ar.ptr(has) : nullptr, ar.ptr(err));
    } else {
        const int32_t* d_ids = ar.put(ids, res->node_id);
        const int32_t* d_oids = tab ? ar.put(oids, res->overhead_node_id) : nullptr;
        ar.fill(rdir, odir, 0xff);
        if (tab) ar.fill(acc, warned, 0);
        GP_TRY(ar.check(c));
        int* e = ar.ptr(err);
        gp_resident_dirs<<<(n + T - 1) / T, T, 0, st>>>(n, d_ids, c->rt.size.n_node_ids, ar.ptr(rdir), d_oids, c->oht.size.n_node_ids,
                                                        ar.ptr(odir), e);
        if (tab) oht_enqueue_sums(c, st, ar.ptr(odir), n, ar.ptr(acc), ar.ptr(warned), ar.ptr(over), nullptr, e + 1);
        const RtCols tc = rt_cols(c);
        if (S)
            gp_usage_scatter<<<(unsigned)((S + T - 1) / T), T, 0, st>>>((long long)S, UsageSlotDir{tc.node, ar.ptr(rdir)}, tc.v[0], tc.v[1],
                                                                       tc.v[2], n, ar.ptr(usage), d_resched ? ar.ptr(has) : nullptr, ar.ptr(err));
    }
    gp_availability<<<(n + T - 1) / T, T, 0, st>>>(n, al[0], al[1], al[2], ov[0], ov[1], ov[2], ar.ptr(usage), ar.ptr(avail), ar.ptr(sched),
                                                   ar.ptr(err), ar.ptr(has), d_resched ? ar.ptr(resched) : nullptr);
    if (d_resched) *d_resched = ar.ptr(resched);
    if (d_over) std::copy(ov, ov + 3, d_over);
    GP_CUDA(c, cudaGetLastError());
    *d_avail = ar.ptr(avail);
    *d_sched = ar.ptr(sched);
    *d_err = ar.ptr(err);
    return GP_OK;
}

// The sort's results on the device.  ig: the instance group of each node (NULL: one); n_zones: the stride of the (instance
// group, zone) pairs (1 when zone is NULL); ig_ties: per instance group undefined ties (NULL without ig).
struct SortStage { const int32_t* drv; const int32_t* exe; const int32_t* counts; const int32_t* zone; const int32_t* ig; int32_t n_zones;
                   const int32_t* ig_ties; };

static void launch_label_keys(int nb, const int32_t* cnt, const int32_t* list, const int32_t* rank, const int32_t*, LabelKey* lk,
                              cudaStream_t st) {
    gp_label_keys<<<nb, 256, 0, st>>>(cnt, list, rank, lk);
}
static void launch_label_keys(int nb, const int32_t* cnt, const int32_t* list, const int32_t* rank, const int32_t* seg, SegLabelKey* lk,
                              cudaStream_t st) {
    gp_seg_label_keys<<<nb, 256, 0, st>>>(cnt, list, rank, seg, lk);
}

// Stable re-sort of list[0..*cnt) by rank[node] (-1 last): out[k] = the k-th node in (rank, position) order.  The label
// re-sort of PotentialNodes, and the zone partition of gp_prepare_cluster_zones.  K = SegLabelKey: by (seg[node], rank,
// position), the label re-sort of an instance-group-major list.
template <class K>
static void launch_label_resort(int32_t n, const int32_t* cnt, const int32_t* list, const int32_t* rank, K* lk, K* lks, int32_t* pos,
                                int32_t* out, cudaStream_t st, const int32_t* seg = nullptr) {
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    launch_label_keys(nb, cnt, list, rank, seg, lk, st);
    gp_sort_tiles<K><<<ntile, kSortThreads, kSortTile * sizeof(K), st>>>(n, cnt, lk, lks);
    gp_rank_by_search<K><<<nb, T, 0, st>>>(n, cnt, lk, lks, pos);
    gp_label_scatter<<<nb, T, 0, st>>>(cnt, list, pos, out);
}

// f1 stage: d_cpu / d_mem / d_gpu are device arrays (NULL: uploaded from `in`; gpu optional); leaves the two orders,
// counts[3] = {#driver candidates, #executor candidates, #undefined ties} and the zone ids (NULL: one zone) on the device.
// ig (host, [n_nodes] in [-1, n_ig), or NULL): PotentialNodes per instance group, instance-group-major (the instance group
// is the leading key; nodes in none are dropped).  The caller has run check_sort_ids and checked ig.  dev: ig and the columns
// of `in` other than is_driver_candidate are device pointers (UsageIn::on_device).
static gp_status stage_sort(gp_ctx* c, const gp_sort_input* in, const int32_t* ig, int32_t n_ig, const long long* d_cpu, const long long* d_mem,
                            const long long* d_gpu, cudaStream_t st, SortStage* out, bool dev = false) {
    const int32_t n = in->n_nodes;
    const bool zoned = in->zone_id != nullptr && in->n_zones > 1;       // one zone: priority 0 for every node, nothing to total
    // one scratch block; the zone totals and priorities are per (instance group, zone) pair
    const int32_t nzk = zoned ? in->n_zones : 1;
    const size_t N = (size_t)n, P = (size_t)n_ig * (size_t)nzk, NI = ig ? N : 0;
    const bool seg_labels = ig && (in->driver_label_rank || in->executor_label_rank);
    Arena ar{c->sortbuf, st};
    const auto cpu = ar.take<long long>(N), mem = ar.take<long long>(N), gpu = ar.take<long long>(N);
    const auto keys = ar.take<SortKey>(N), sorted = ar.take<SortKey>(N);
    const auto tot = ar.take<unsigned long long>(kZoneTotWords * P);
    const auto zone = ar.take<int32_t>(N), nr = ar.take<int32_t>(N), prio = ar.take<int32_t>(P), pos = ar.take<int32_t>(N),
               order = ar.take<int32_t>(N), drv = ar.take<int32_t>(N), exe = ar.take<int32_t>(N), drv2 = ar.take<int32_t>(N),
               exe2 = ar.take<int32_t>(N), lrd = ar.take<int32_t>(N), lre = ar.take<int32_t>(N);
    const auto lk = ar.take<LabelKey>(seg_labels ? 0 : N), lks = ar.take<LabelKey>(seg_labels ? 0 : N);
    const auto slk = ar.take<SegLabelKey>(seg_labels ? N : 0), slks = ar.take<SegLabelKey>(seg_labels ? N : 0);
    const auto cnt = ar.take<int32_t>(4);
    const auto fc = ar.take<uint8_t>(N), fu = ar.take<uint8_t>(N), fr = ar.take<uint8_t>(N);
    const auto igp = ar.take<int32_t>(NI), ties = ar.take<int32_t>(ig ? (size_t)n_ig : 0);
    ar.reserve();
    if (!d_cpu) d_cpu = ar.put(cpu, in->avail_cpu_milli);
    if (!d_mem) d_mem = ar.put(mem, in->avail_mem_bytes);
    if (!d_gpu) d_gpu = ar.put(gpu, in->avail_gpu);
    const int32_t* d_zone = !zoned ? nullptr : dev ? in->zone_id : ar.put(zone, in->zone_id);
    const int32_t* d_ig = dev ? ig : ar.put(igp, ig);
    int32_t* d_ties = ig ? ar.zero(ties) : nullptr;
    const int32_t* d_nr = dev ? in->name_rank : ar.put(nr, in->name_rank);
    const uint8_t* d_fc = ar.put(fc, in->is_driver_candidate);
    const uint8_t* d_fu = dev ? in->unschedulable : ar.put(fu, in->unschedulable);
    const uint8_t* d_fr = dev ? in->ready : ar.put(fr, in->ready);
    const int32_t* d_lrd = dev ? in->driver_label_rank : ar.put(lrd, in->driver_label_rank);
    const int32_t* d_lre = dev ? in->executor_label_rank : ar.put(lre, in->executor_label_rank);
    if (zoned) ar.zero(tot);
    GP_TRY(ar.check(c));
    if (!c->sort_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<SortKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(SortKey))));
        c->sort_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    if (zoned) {
        gp_zone_totals<<<nb, T, 0, st>>>(n, d_cpu, d_mem, d_zone, d_ig, nzk, ar.ptr(tot));
        gp_zone_priority<<<(unsigned)((P + T - 1) / T), T, 0, st>>>((int32_t)P, nzk, ar.ptr(tot), ar.ptr(prio));
    }
    gp_make_keys<<<nb, T, 0, st>>>(n, d_cpu, d_mem, d_zone, ar.ptr(prio), d_ig, n_ig, nzk, d_nr, ar.ptr(keys));
    gp_sort_tiles<SortKey><<<ntile, kSortThreads, kSortTile * sizeof(SortKey), st>>>(n, nullptr, ar.ptr(keys), ar.ptr(sorted));
    gp_rank_by_search<SortKey><<<nb, T, 0, st>>>(n, nullptr, ar.ptr(keys), ar.ptr(sorted), ar.ptr(pos));
    gp_scatter_order<<<nb, T, 0, st>>>(n, ar.ptr(pos), ar.ptr(order));
    if (d_ig) gp_split_candidates<true><<<1, 1024, 0, st>>>(n, ar.ptr(order), d_fc, d_fu, d_fr, ar.ptr(keys), d_gpu, d_ig, d_ties, ar.ptr(drv),
                                                            ar.ptr(exe), ar.ptr(cnt));
    else gp_split_candidates<false><<<1, 1024, 0, st>>>(n, ar.ptr(order), d_fc, d_fu, d_fr, ar.ptr(keys), d_gpu, nullptr, nullptr, ar.ptr(drv),
                                                        ar.ptr(exe), ar.ptr(cnt));
    out->drv = ar.ptr(drv);
    out->exe = ar.ptr(exe);
    out->counts = ar.ptr(cnt);
    out->zone = d_zone;
    out->ig = d_ig;
    out->n_zones = nzk;
    out->ig_ties = d_ties;
    auto label_sort = [&](const int32_t* count, const int32_t* list, const int32_t* rank, Piece<int32_t> to) {
        if (seg_labels) launch_label_resort(n, count, list, rank, ar.ptr(slk), ar.ptr(slks), ar.ptr(pos), ar.ptr(to), st, d_ig);
        else launch_label_resort(n, count, list, rank, ar.ptr(lk), ar.ptr(lks), ar.ptr(pos), ar.ptr(to), st);
        return (const int32_t*)ar.ptr(to);
    };
    if (d_lrd) out->drv = label_sort(out->counts, out->drv, d_lrd, drv2);
    if (d_lre) out->exe = label_sort(out->counts + 1, out->exe, d_lre, exe2);
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// gp_prepare_cluster and gp_prepare_cluster_zones up to their layout step: the checks both make, then reservations ->
// availability (d_avail / d_sched: [3][n_nodes]) -> priority orders on the context's stream.  Synchronises once for the
// availability stage's status word: a refusal returns before anything of the context's snapshot has been replaced.
// ig / n_ig: the instance groups of stage_sort, already checked.
static gp_status prepare_orders(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* ig, int32_t n_ig,
                                const char* who, long long** d_avail, long long** d_sched, SortStage* so) {
    GP_TRY(check_source(c, usage, who));
    if (!sort || usage.n_nodes() != sort->n_nodes || sort->n_zones < 1)
        return fail(c, GP_ERR_INVALID, who, "missing arrays or mismatched sizes");
    if (usage.n_nodes() == 0) return fail(c, GP_ERR_INVALID, who, "empty node table");
    if (!usage.on_device()) GP_TRY(check_sort_ids(c, sort, who));
    GP_CUDA(c, cudaSetDevice(c->device));
    int* d_err = nullptr;
    GP_TRY(stage_availability(c, usage, c->stream, d_avail, d_sched, &d_err));
    const size_t N = (size_t)usage.n_nodes();
    GP_TRY(stage_sort(c, sort, ig, n_ig, *d_avail, *d_avail + N, *d_avail + 2 * N, c->stream, so, usage.on_device()));
    int err[2] = {0, 0}, gather = 0;
    GP_CUDA(c, cudaMemcpyAsync(err, d_err, sizeof err, cudaMemcpyDeviceToHost, c->stream));
    if (usage.on_device()) GP_CUDA(c, cudaMemcpyAsync(&gather, usage.gather_err, sizeof gather, cudaMemcpyDeviceToHost, c->stream));
    GP_CUDA(c, cudaStreamSynchronize(c->stream));
    GP_TRY(nt_refusal(c, gather, who));
    return stage_refusal(c, err, who);
}

// gp_prepare_cluster and gp_prepare_cluster_zones after their layout step, which set dn's groups, offsets and orders: the
// node-table copy (gp_get_snapshot), the usual slot layout with n_nodes bounding both order lengths, SchedulableResources,
// and counts[3] of the sort read back (the caller synchronises).
static gp_status prepare_snapshot(gp_ctx* c, gp_nodes* dn, const long long* d_avail, const long long* d_sched, const SortStage& so,
                                  int32_t* counts) {
    cudaStream_t st = c->stream;
    const int32_t n = dn->n_nodes;
    const size_t N = (size_t)n, nb = sizeof(int64_t) * (N + 1);
    GP_CUDA(c, c->node_cpu.reserve(nb)); GP_CUDA(c, c->node_mem.reserve(nb)); GP_CUDA(c, c->node_gpu.reserve(nb));
    GP_CUDA(c, cudaMemcpyAsync(c->node_cpu.p, d_avail, 8 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(c->node_mem.p, d_avail + N, 8 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(c->node_gpu.p, d_avail + 2 * N, 8 * N, cudaMemcpyDeviceToDevice, st));
    dn->avail_cpu_milli = c->node_cpu.as<int64_t>(); dn->avail_mem_bytes = c->node_mem.as<int64_t>(); dn->avail_gpu = c->node_gpu.as<int64_t>();
    gp_status s = build_snapshot_device(c, dn, n, n, st);
    if (s != GP_OK) return s;
    GP_CUDA(c, c->sched.reserve(24 * (N + 1)));
    GP_CUDA(c, cudaMemcpyAsync(c->sched.p, d_sched, 24 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(counts, so.counts, 12, cudaMemcpyDeviceToHost, st));
    return GP_OK;
}

// The instance-group arguments of gp_prepare_cluster_groups and gp_prepare_cluster_zones_groups: n_ig >= 1, values in
// [-1, n_ig), and with several instance groups at most 2^22 (instance group, zone + 1) pairs (stage_sort's zone totals are
// per pair).  The other arguments are checked by prepare_orders.
static gp_status check_instance_groups(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* ig, int32_t n_ig,
                                       const char* who) {
    if (n_ig < 1) return fail(c, GP_ERR_INVALID, who, "n_instance_groups must be >= 1");
    if (sort && n_ig > 1 && (int64_t)n_ig * ((int64_t)sort->n_zones + 1) > kZoneLayoutMaxPairs)
        return fail(c, GP_ERR_INVALID, who, "n_instance_groups x (n_zones + 1) above 2^22");
    if (ig && usage.given() && !usage.on_device() && sort && usage.n_nodes() == sort->n_nodes)
        for (int32_t i = 0; i < usage.n_nodes(); ++i)
            if (ig[i] < -1 || ig[i] >= n_ig) return fail(c, GP_ERR_INVALID, who, "instance_group outside [-1, n_instance_groups)");
    return GP_OK;
}

// gp_prepare_cluster (ig NULL, n_ig 1) and gp_prepare_cluster_groups: the checks, reservations -> availability ->
// instance-group-major priority orders (prepare_orders, which synchronises once and refuses before anything of the context
// is replaced) -> snapshot group g = instance group g's range of those orders (gp_ig_offsets) -> the slot layout, then one
// synchronise that reads back counts[3] and, when ig_ties is given, the undefined ties [n_ig] of each instance group.
// ig NULL with n_ig > 1: every node in instance group 0, the others empty.
static gp_status prepare_groups(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* ig, int32_t n_ig,
                                const char* who, int32_t* counts, int32_t* ig_ties, SortStage* so_out = nullptr) {
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    GP_TRY(prepare_orders(c, usage, sort, ig, ig ? n_ig : 1, who, &d_avail, &d_sched, &so));
    c->held.commit();
    cudaStream_t st = c->stream;
    const size_t G1 = (size_t)n_ig + 1;
    GP_CUDA(c, c->exec_off.reserve(4 * G1)); GP_CUDA(c, c->drv_off.reserve(4 * G1));
    const int T = 256;
    gp_ig_offsets<<<(unsigned)((G1 + T - 1) / T), T, 0, st>>>(n_ig, so.counts, so.drv, so.exe, so.ig, c->exec_off.as<int32_t>(),
                                                               c->drv_off.as<int32_t>());
    GP_CUDA(c, cudaGetLastError());
    gp_nodes dn{};
    dn.n_nodes = usage.n_nodes();
    dn.n_groups = n_ig;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = so.exe;
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = so.drv;
    GP_TRY(prepare_snapshot(c, &dn, d_avail, d_sched, so, counts));
    if (ig_ties && so.ig_ties) GP_CUDA(c, cudaMemcpyAsync(ig_ties, so.ig_ties, 4 * (size_t)n_ig, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (ig_ties && !so.ig_ties) {                       // one instance group holds every node: its ties are the total
        std::fill(ig_ties, ig_ties + n_ig, 0);
        ig_ties[0] = counts[2];
    }
    c->n_drv = counts[0]; c->n_exec = counts[1];
    c->held.laid_out_cluster();
    if (sort->undefined_ties) *sort->undefined_ties = counts[2];
    if (so_out) *so_out = so;
    return GP_OK;
}

// The two gp_build_*availability entries: the availability stage, then every non-NULL outs[k] gets row k % 3 of
// availableResources for k < 3 (first_fit: that of rescheduleExecutor's first-fit branch), of SchedulableResources for k >= 3.
// The stage's status word is read first: a refused call writes to none of them.
static gp_status availability_out(gp_ctx* c, const gp_usage_input* in, bool first_fit, int64_t* const* outs, const char* who) {
    gp_status s = check_usage(c, in, who);
    if (s != GP_OK) return s;
    const int32_t n = in->n_nodes;
    if (n == 0) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    long long *d_avail = nullptr, *d_sched = nullptr, *d_ff = nullptr;
    int* d_err = nullptr;
    s = stage_availability(c, in, st, &d_avail, &d_sched, &d_err, first_fit ? &d_ff : nullptr);
    if (s != GP_OK) return s;
    int err = 0;
    GP_CUDA(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    GP_TRY(refuse(c, err, kFeRefusals, who));                           // the outputs are left as they were
    const size_t N = (size_t)n;
    const long long* src[2] = {first_fit ? d_ff : d_avail, d_sched};
    for (int k = 0; k < 6; ++k)
        if (outs[k]) GP_CUDA(c, cudaMemcpyAsync(outs[k], src[k / 3] + N * (size_t)(k % 3), 8 * N, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

// What prepare_zones leaves for its entry: the sort's counts[3], the ZoneInfo words, the device zone_of_group, the IgWords read back.
struct ZonePrep {
    int32_t counts[3];
    int32_t info[kZiWords];
    const int32_t* zone_of_group;
    std::vector<int32_t> ig_words;
};

// gp_prepare_cluster_zones (ig NULL, n_ig 1) and gp_prepare_cluster_zones_groups up to their optional outputs: the checks,
// reservations -> availability -> instance-group-major priority orders (prepare_orders, which synchronises once and refuses
// before anything of the context is replaced) -> the zone-grouped layout (gangpack_zonelayout.cuh) -> the slot layout, then
// one synchronise that reads back the counts.  zog_now (or NULL): zone_of_group [sort->n_zones + 1] read back in that
// synchronise; ig_ties (or NULL): the undefined ties [n_ig] likewise.  keep_ig (gp_prepare_cluster_zones_groups): the
// per-instance-group words are held (Held::groups).  ig NULL with n_ig > 1: every node in instance group 0, the others empty.
static gp_status prepare_zones(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* ig, int32_t n_ig,
                               int32_t kind, bool keep_ig, const char* who, int32_t* zog_now, int32_t* ig_ties, ZonePrep* zp) {
    if (kind != GP_LAYOUT_SINGLE_AZ && kind != GP_LAYOUT_AZ_AWARE)
        return fail(c, GP_ERR_INVALID, who, "layout->kind must be GP_LAYOUT_SINGLE_AZ or GP_LAYOUT_AZ_AWARE");
    if (sort && sort->n_zones == 0x7fffffff) return fail(c, GP_ERR_INVALID, who, "n_zones too large");
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    GP_TRY(prepare_orders(c, usage, sort, ig, n_ig, who, &d_avail, &d_sched, &so));
    c->held.commit();                                   // the held orders are overwritten below
    cudaStream_t st = c->stream;
    const int32_t n = usage.n_nodes();
    const size_t N = (size_t)n, G1 = (size_t)n_ig + 1;
    // the (instance group, zone) pairs; g_bound groups bound every layout (each instance group: its candidate zones plus
    // one; a candidate zone holds a node).  The slots are laid out for that many (the groups past the last one are empty)
    // so that the group count can stay on the device until the one synchronise below.
    const size_t P = (size_t)n_ig * (size_t)so.n_zones;
    const int32_t g_bound = (int32_t)std::min<int64_t>((int64_t)P + n_ig, (int64_t)n + n_ig);
    Arena ar{c->zoneprep, st};
    const auto udrv_p = ar.take<int32_t>(N), uexe_p = ar.take<int32_t>(N), first = ar.take<int32_t>(P);
    const auto has = ar.take<uint8_t>(P);
    const auto zg = ar.take<int32_t>(P), zog = ar.take<int32_t>(std::max<size_t>((size_t)g_bound, (size_t)sort->n_zones + 1)),
               rank_p = ar.take<int32_t>(N);
    const auto lk = ar.take<LabelKey>(N), lks = ar.take<LabelKey>(N);
    const auto pos = ar.take<int32_t>(N), info_p = ar.take<int32_t>(kZiWords), igw = ar.take<int32_t>(6 * G1);
    ar.reserve();
    GP_TRY(ar.check(c));
    int32_t* udrv = ar.ptr(udrv_p);
    int32_t* uexe = ar.ptr(uexe_p);
    int32_t* info = ar.ptr(info_p);
    int32_t* rank = ar.ptr(rank_p);
    int32_t* wb = ar.ptr(igw);
    // group_off, n_zones, exec_off, drv_off adjacent: the host copy is one read
    const IgWords w{wb + G1, wb + 4 * G1, wb, wb + 5 * G1, wb + 2 * G1, wb + 3 * G1};
    // the undivided orders outlive the sort's scratch, which the next gp_potential_nodes / gp_prepare_cluster reuses
    GP_CUDA(c, cudaMemcpyAsync(udrv, so.drv, 4 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(uexe, so.exe, 4 * N, cudaMemcpyDeviceToDevice, st));
    ar.fill(first, 0x7f);
    ar.zero(has);
    ar.fill(zg, zog, 0xff);
    ar.fill(info_p, igw, 0);
    GP_TRY(ar.check(c));
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int32_t az = kind == GP_LAYOUT_AZ_AWARE ? 1 : 0;
    gp_zone_mark<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, so.ig, so.n_zones, ar.ptr(first), ar.ptr(has));
    gp_zone_candidates<<<1, 1024, 0, st>>>(so.counts, udrv, so.zone, so.ig, so.n_zones, n_ig, az, ar.ptr(first), ar.ptr(has), ar.ptr(zg),
                                           ar.ptr(zog), w, info);
    gp_group_rank<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, so.ig, so.n_zones, ar.ptr(zg), az, w, rank);
    GP_CUDA(c, cudaGetLastError());
    // the grouped orders and their offsets
    GP_CUDA(c, c->exec_order.reserve(4 * (N + 1))); GP_CUDA(c, c->drv_order.reserve(4 * (N + 1)));
    GP_CUDA(c, c->exec_off.reserve(4 * ((size_t)g_bound + 1))); GP_CUDA(c, c->drv_off.reserve(4 * ((size_t)g_bound + 1)));
    launch_label_resort(n, so.counts, udrv, rank, ar.ptr(lk), ar.ptr(lks), ar.ptr(pos), c->drv_order.as<int32_t>(), st);
    launch_label_resort(n, so.counts + 1, uexe, rank, ar.ptr(lk), ar.ptr(lks), ar.ptr(pos), c->exec_order.as<int32_t>(), st);
    gp_group_offsets<<<(unsigned)((g_bound + T) / T), T, 0, st>>>(g_bound, so.counts, c->drv_order.as<int32_t>(), c->exec_order.as<int32_t>(),
                                                                  rank, az, c->exec_off.as<int32_t>(), c->drv_off.as<int32_t>(), info, n_ig,
                                                                  so.ig, udrv, uexe, w);
    GP_CUDA(c, cudaGetLastError());
    gp_nodes dn{};
    dn.n_nodes = n;
    dn.n_groups = g_bound;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = c->exec_order.as<int32_t>();
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = c->drv_order.as<int32_t>();
    GP_TRY(prepare_snapshot(c, &dn, d_avail, d_sched, so, zp->counts));
    ar.get(zp->info, info_p);
    ar.get(zog_now, zog.part(0, (size_t)sort->n_zones + 1));
    zp->ig_words.resize(4 * G1);
    ar.get(zp->ig_words.data(), wb, 4 * G1);
    if (so.ig_ties) ar.get(ig_ties, so.ig_ties, (size_t)n_ig);
    GP_TRY(ar.sync(c));
    if (!so.ig_ties && ig_ties) {                       // one instance group holds every node: its ties are the total
        std::fill(ig_ties, ig_ties + n_ig, 0);
        ig_ties[0] = zp->counts[2];
    }
    c->n_groups = zp->info[kZiGroups]; c->n_exec = zp->info[kZiExec]; c->n_drv = zp->info[kZiDrv];
    c->held.laid_out_zones(kind, gp_az_orders{zp->info[kZiZones], zp->counts[1], uexe, zp->counts[0], udrv}, keep_ig ? n_ig : 0, zp->ig_words.data());
    zp->zone_of_group = ar.ptr(zog);
    return GP_OK;
}

extern "C" {

gp_status gp_potential_nodes(gp_ctx* c, const gp_sort_input* in, int32_t* driver_order, int32_t* n_driver,
                             int32_t* executor_order, int32_t* n_executor) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!in || in->n_nodes < 0 || in->n_zones < 1 || !n_driver || !n_executor ||
        (in->n_nodes > 0 && (!in->avail_cpu_milli || !in->avail_mem_bytes || !driver_order || !executor_order)))
        return fail(c, GP_ERR_INVALID, "gp_potential_nodes: missing arrays or bad sizes");
    const int32_t n = in->n_nodes;
    *n_driver = 0; *n_executor = 0;
    if (n == 0) return GP_OK;
    gp_status s = check_sort_ids(c, in, "gp_potential_nodes");
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    SortStage so{};
    s = stage_sort(c, in, nullptr, 1, nullptr, nullptr, nullptr, st, &so);
    if (s != GP_OK) return s;
    int32_t counts[3] = {0, 0, 0};
    GP_CUDA(c, cudaMemcpyAsync(counts, so.counts, 12, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(driver_order, so.drv, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(executor_order, so.exe, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    *n_driver = counts[0];
    *n_executor = counts[1];
    if (in->undefined_ties) *in->undefined_ties = counts[2];
    return GP_OK;
}

gp_status gp_build_availability(gp_ctx* c, const gp_usage_input* in, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu,
                                int64_t* sched_cpu, int64_t* sched_mem, int64_t* sched_gpu) {
    if (!enter(c)) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, sched_cpu, sched_mem, sched_gpu};
    return availability_out(c, in, false, outs, "gp_build_availability");
}

// availableResources of rescheduleExecutor's first-fit branch: the availability to upload before gp_reschedule_executors(min_frag = 0)
gp_status gp_build_reschedule_availability(gp_ctx* c, const gp_usage_input* in, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu) {
    if (!enter(c)) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, nullptr, nullptr, nullptr};
    return availability_out(c, in, true, outs, "gp_build_reschedule_availability");
}

// reservations -> availability -> priority orders -> slot layout, without leaving the device
gp_status gp_prepare_cluster(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, int32_t* n_driver, int32_t* n_executor) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (n_driver) *n_driver = 0;
    if (n_executor) *n_executor = 0;
    int32_t counts[3] = {0, 0, 0};
    GP_TRY(prepare_groups(c, usage, sort, nullptr, 1, "gp_prepare_cluster", counts, nullptr));
    if (n_driver) *n_driver = counts[0];
    if (n_executor) *n_executor = counts[1];
    return GP_OK;
}

}  // extern "C"

// gp_prepare_cluster_groups[_resident]
static gp_status prepare_cluster_groups(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* instance_group,
                                        int32_t n_instance_groups, gp_instance_group_orders* out, const char* who) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!out) return fail(c, GP_ERR_INVALID, who, "missing arrays or mismatched sizes");
    out->n_driver = 0; out->n_executor = 0;
    const int32_t G = n_instance_groups;
    GP_TRY(check_instance_groups(c, usage, sort, instance_group, G, who));
    int32_t counts[3] = {0, 0, 0};
    SortStage so{};
    GP_TRY(prepare_groups(c, usage, sort, instance_group, G, who, counts, out->undefined_ties, &so));
    out->n_driver = counts[0]; out->n_executor = counts[1];
    // the orders and their offsets only when asked: the snapshot's own exec_off / drv_off, and the sort's orders, which stay
    // in its scratch until the next sort
    Arena ar{c->zoneprep, c->stream};
    const size_t g1 = (size_t)G + 1;
    ar.get(out->exec_off, c->exec_off.as<int32_t>(), g1);
    ar.get(out->drv_off, c->drv_off.as<int32_t>(), g1);
    ar.get(out->exec_order, so.exe, (size_t)counts[1]);
    ar.get(out->drv_order, so.drv, (size_t)counts[0]);
    if (out->exec_off || out->drv_off || out->exec_order || out->drv_order) GP_TRY(ar.sync(c));
    return GP_OK;
}

extern "C" {

// the same chain for every instance group at once: snapshot group i holds instance group i's PotentialNodes orders
gp_status gp_prepare_cluster_groups(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const int32_t* instance_group,
                                    int32_t n_instance_groups, gp_instance_group_orders* out) {
    return prepare_cluster_groups(c, usage, sort, instance_group, n_instance_groups, out, "gp_prepare_cluster_groups");
}

// the same with the reservations (and optionally the overhead) from the context's resident tables
gp_status gp_prepare_cluster_groups_resident(gp_ctx* c, const gp_resident_usage* usage, const gp_sort_input* sort,
                                             const int32_t* instance_group, int32_t n_instance_groups, gp_instance_group_orders* out) {
    return prepare_cluster_groups(c, usage, sort, instance_group, n_instance_groups, out, "gp_prepare_cluster_groups_resident");
}

// reservations -> availability -> priority orders -> zone-grouped slot layout, without leaving the device
gp_status gp_prepare_cluster_zones(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, gp_zone_layout* layout) {
    const char* who = "gp_prepare_cluster_zones";
    if (!enter(c)) return GP_ERR_INVALID;
    if (!layout) return fail(c, GP_ERR_INVALID, who, "missing arrays or mismatched sizes");
    layout->n_zones = 0; layout->n_groups = 0; layout->n_driver = 0; layout->n_executor = 0;
    ZonePrep zp{};
    GP_TRY(prepare_zones(c, usage, sort, nullptr, 1, layout->kind, false, who, layout->zone_of_group, nullptr, &zp));
    if (sort->undefined_ties) *sort->undefined_ties = zp.counts[2];
    layout->n_zones = zp.info[kZiZones]; layout->n_groups = zp.info[kZiGroups];
    layout->n_driver = zp.counts[0]; layout->n_executor = zp.counts[1];
    // the grouped layout itself only when asked: its sizes are known now
    Arena ar{c->zoneprep, c->stream};
    const size_t n_off = (size_t)zp.info[kZiGroups] + 1;
    ar.get(layout->exec_off, c->exec_off.as<int32_t>(), n_off);
    ar.get(layout->drv_off, c->drv_off.as<int32_t>(), n_off);
    ar.get(layout->exec_order, c->exec_order.as<int32_t>(), (size_t)c->n_exec);
    ar.get(layout->drv_order, c->drv_order.as<int32_t>(), (size_t)c->n_drv);
    if (layout->exec_off || layout->drv_off || layout->exec_order || layout->drv_order) GP_TRY(ar.sync(c));
    return GP_OK;
}

}  // extern "C"

// gp_prepare_cluster_zones_groups[_resident]
static gp_status prepare_cluster_zones_groups(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const int32_t* instance_group,
                                              int32_t n_instance_groups, gp_instance_group_layout* layout, const char* who) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!layout) return fail(c, GP_ERR_INVALID, who, "missing arrays or mismatched sizes");
    layout->n_groups = 0; layout->n_driver = 0; layout->n_executor = 0;
    const int32_t G = n_instance_groups;
    GP_TRY(check_instance_groups(c, usage, sort, instance_group, G, who));
    ZonePrep zp{};
    GP_TRY(prepare_zones(c, usage, sort, instance_group, G, layout->kind, true, who, nullptr, layout->undefined_ties, &zp));
    if (sort->undefined_ties) *sort->undefined_ties = zp.counts[2];
    const int32_t n_groups = zp.info[kZiGroups];
    layout->n_groups = n_groups; layout->n_driver = zp.counts[0]; layout->n_executor = zp.counts[1];
    // the per-instance-group words are on the host already; the rest only when asked
    const size_t g1 = (size_t)G + 1;
    const gp_instance_groups held = c->held.groups();
    if (layout->group_off) std::copy(held.group_off, held.group_off + g1, layout->group_off);
    if (layout->n_zones) std::copy(held.n_zones, held.n_zones + G, layout->n_zones);
    if (layout->exec_off) std::copy(held.exec_off, held.exec_off + g1, layout->exec_off);
    if (layout->drv_off) std::copy(held.drv_off, held.drv_off + g1, layout->drv_off);
    Arena ar{c->zoneprep, c->stream};
    const size_t n_off = (size_t)n_groups + 1;
    ar.get(layout->exec_order, held.exec_order, (size_t)zp.counts[1]);
    ar.get(layout->drv_order, held.drv_order, (size_t)zp.counts[0]);
    ar.get(layout->group_exec_off, c->exec_off.as<int32_t>(), n_off);
    ar.get(layout->group_drv_off, c->drv_off.as<int32_t>(), n_off);
    ar.get(layout->group_exec_order, c->exec_order.as<int32_t>(), (size_t)c->n_exec);
    ar.get(layout->group_drv_order, c->drv_order.as<int32_t>(), (size_t)c->n_drv);
    ar.get(layout->zone_of_group, zp.zone_of_group, (size_t)n_groups);
    if (layout->exec_order || layout->drv_order || layout->group_exec_off || layout->group_drv_off || layout->group_exec_order ||
        layout->group_drv_order || layout->zone_of_group)
        GP_TRY(ar.sync(c));
    return GP_OK;
}

extern "C" {

// the same chain for every instance group at once: the layout of each one is gp_prepare_cluster_zones' on its nodes alone
gp_status gp_prepare_cluster_zones_groups(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const int32_t* instance_group,
                                          int32_t n_instance_groups, gp_instance_group_layout* layout) {
    return prepare_cluster_zones_groups(c, usage, sort, instance_group, n_instance_groups, layout, "gp_prepare_cluster_zones_groups");
}

// the same with the reservations (and optionally the overhead) from the context's resident tables
gp_status gp_prepare_cluster_zones_groups_resident(gp_ctx* c, const gp_resident_usage* usage, const gp_sort_input* sort,
                                                   const int32_t* instance_group, int32_t n_instance_groups, gp_instance_group_layout* layout) {
    return prepare_cluster_zones_groups(c, usage, sort, instance_group, n_instance_groups, layout, "gp_prepare_cluster_zones_groups_resident");
}

// rescheduleExecutor's node choice for a batch of executors (SURVEY 8f row f4); see gangpack_resched.cuh
gp_status gp_reschedule_executors(gp_ctx* c, const gp_reschedule* in, int32_t* node_out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), "gp_reschedule_executors"));
    if (!in || in->n_execs < 0 || (in->n_execs > 0 && (!in->exe_cpu_milli || !in->exe_mem_bytes || !node_out)))
        return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: missing arrays or bad sizes");
    const int32_t q = in->n_execs;
    if (q == 0) return GP_OK;
    const bool mf = in->min_frag != 0;
    const bool has_res = mf && in->reserved_cpu_milli;
    const bool has_host = mf && in->host_off;
    if (has_res && !in->reserved_mem_bytes) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: reserved_mem_bytes missing");
    // host validation (O(q + n_nodes + hosted)): the exact-int64 domain, non-negative requests, CSR shape
    gp_status chk = check_requests(c, q, in->exe_cpu_milli, in->exe_mem_bytes, in->exe_gpu, "gp_reschedule_executors");
    if (chk != GP_OK) return chk;
    for (int32_t i = 0; i < q; ++i)
        if (in->group && (in->group[i] < 0 || in->group[i] >= c->n_groups)) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: instance group out of range");
    if (has_res)
        for (int32_t n = 0; n < c->n_nodes; ++n) {
            const int64_t v[3] = {in->reserved_cpu_milli[n], in->reserved_mem_bytes[n], in->reserved_gpu ? in->reserved_gpu[n] : 0};
            for (int64_t x : v)
                if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_reschedule_executors: |reserved| >= 2^61");
        }
    int64_t hosted = 0;
    if (has_host && (chk = check_hosting(c, in, c->n_nodes, &hosted, "gp_reschedule_executors")) != GP_OK) return chk;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t Q = (size_t)q, N = (size_t)c->n_nodes, H = (size_t)hosted;
    Arena ar{c->callbuf, st};
    const auto exe = ar.take<int64_t>(3 * Q), res = ar.take<int64_t>(3 * N), hoff = ar.take<int64_t>(Q + 1);
    const auto grp = ar.take<int32_t>(Q), hn = ar.take<int32_t>(H + 1), d_out = ar.take<int32_t>(Q);
    const auto d_err = ar.take<int>(2);
    ar.reserve();
    ar.zero(d_err);
    ReschedIn ri{};
    ri.exe_cpu = ar.put(exe.part(0, Q), in->exe_cpu_milli);
    ri.exe_mem = ar.put(exe.part(Q, Q), in->exe_mem_bytes);
    ri.exe_gpu = ar.put(exe.part(2 * Q, Q), in->exe_gpu);
    ri.group = ar.put(grp, in->group);
    if (has_res) {
        ri.res_cpu = ar.put(res.part(0, N), in->reserved_cpu_milli);
        ri.res_mem = ar.put(res.part(N, N), in->reserved_mem_bytes);
        ri.res_gpu = ar.put(res.part(2 * N, N), in->reserved_gpu);
    }
    if (has_host) {
        ri.host_off = ar.put(hoff, in->host_off);
        ar.put(hn.part(0, H), in->host_nodes);
    }
    ri.host_nodes = ar.ptr(hn);
    ri.node_slot = c->node_slot.as<int32_t>();
    ri.n_execs = q;
    const Snapshot s = make_snapshot(c);
    const int T = 256;
    int64_t blocks = ((int64_t)q * 32 + T - 1) / T;
    const int64_t max_blocks = (int64_t)c->sm_count * 8;
    if (blocks > max_blocks) blocks = max_blocks;
    GP_TRY(ar.check(c));
    if (mf) gp_reschedule_kernel<true><<<(int)blocks, T, 0, st>>>(s, ri, ar.ptr(d_out), ar.ptr(d_err));
    else gp_reschedule_kernel<false><<<(int)blocks, T, 0, st>>>(s, ri, ar.ptr(d_out), ar.ptr(d_err));
    GP_CUDA(c, cudaGetLastError());
    int err = 0;
    ar.get(node_out, d_out);
    ar.get(&err, ar.ptr(d_err), 1);
    GP_TRY(ar.sync(c));
    if (err) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: instance group out of range");
    return GP_OK;
}

}  // extern "C"

// gp_reschedule_from_reservations[_resident]
static gp_status reschedule_from_reservations(gp_ctx* c, const UsageIn& usage, const gp_sort_input* sort, const gp_reschedule_scope* scope,
                                              const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous, const char* who) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(check_source(c, usage, who));
    if (!sort || !in || usage.n_nodes() != sort->n_nodes || sort->n_zones < 1 ||
        in->n_execs < 0 || (in->n_execs > 0 && (!in->exe_cpu_milli || !in->exe_mem_bytes || !node_out)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or mismatched sizes");
    const int32_t n = usage.n_nodes(), q = in->n_execs;
    if (n == 0) return fail(c, GP_ERR_INVALID, who, "empty node table");
    if (in->reserved_cpu_milli || in->reserved_mem_bytes || in->reserved_gpu)
        return fail(c, GP_ERR_INVALID, who, "reserved_* must be NULL (the overhead of the node table is the reserved amount)");
    const int32_t keep = scope ? scope->keep_topology_zone : -1;
    if (keep < -1) return fail(c, GP_ERR_INVALID, who, "scope->keep_topology_zone must be -1 or a zone id");
    if (keep >= 0) {
        if (!scope->topology_zone) return fail(c, GP_ERR_INVALID, who, "scope->topology_zone missing");
        for (int32_t i = 0; i < n; ++i)
            if (scope->topology_zone[i] < 0)
                return fail(c, GP_ERR_INVALID, who, "filterNodesToZone: a node has no topology.kubernetes.io/zone label (topology_zone == -1), "
                                                    "unable to make scheduling decisions based on AZ");
    }
    if (!usage.on_device()) GP_TRY(check_sort_ids(c, sort, who));
    const bool mf = in->min_frag != 0;
    const bool has_host = mf && in->host_off;
    GP_TRY(check_requests(c, q, in->exe_cpu_milli, in->exe_mem_bytes, in->exe_gpu, who));
    for (int32_t i = 0; i < q; ++i)
        if (in->group && in->group[i] != 0) return fail(c, GP_ERR_INVALID, who, "instance group out of range (one node table: group must be 0)");
    int64_t hosted = 0;
    if (has_host) GP_TRY(check_hosting(c, in, n, &hosted, who));
    if (q == 0) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    // availability: one scatter of the reservations, one pass per node (usagebuf is scratch of the f2 stage only)
    long long *d_avail = nullptr, *d_sched = nullptr, *d_ff = nullptr;
    const long long* d_over[3] = {nullptr, nullptr, nullptr};
    int* d_err = nullptr;
    GP_TRY(stage_availability(c, usage, st, &d_avail, &d_sched, &d_err, mf ? nullptr : &d_ff, d_over));
    const size_t N = (size_t)n, Q = (size_t)q, H = (size_t)hosted, Z = (size_t)sort->n_zones;
    const bool zoned = sort->zone_id != nullptr && sort->n_zones > 1;
    Arena ar{c->callbuf, st};
    const auto tot = ar.take<unsigned long long>(kZoneTotWords * Z);
    const auto prio = ar.take<int32_t>(Z), zone = ar.take<int32_t>(N), nr = ar.take<int32_t>(N);
    const auto fu = ar.take<uint8_t>(N), fr = ar.take<uint8_t>(N);
    const auto lr = ar.take<int32_t>(N), tz = ar.take<int32_t>(N);
    const auto rec = ar.take<RpNode>(N);
    const auto exe = ar.take<int64_t>(3 * Q), hoff = ar.take<int64_t>(Q + 1);
    const auto hn = ar.take<int32_t>(H + 1), d_out = ar.take<int32_t>(Q);
    const auto amb = ar.take<uint8_t>(Q);
    ar.reserve();
    RpNodeIn ni{};
    const bool dev = usage.on_device();
    ni.zone = !zoned ? nullptr : dev ? sort->zone_id : ar.put(zone, sort->zone_id);
    ni.name_rank = dev ? sort->name_rank : ar.put(nr, sort->name_rank);
    ni.unschedulable = dev ? sort->unschedulable : ar.put(fu, sort->unschedulable);
    ni.ready = dev ? sort->ready : ar.put(fr, sort->ready);
    ni.label_rank = dev ? sort->executor_label_rank : ar.put(lr, sort->executor_label_rank);
    ni.tz = keep >= 0 ? ar.put(tz, scope->topology_zone) : nullptr;
    RpDecideIn di{};
    di.exe = ar.put(exe.part(0, Q), in->exe_cpu_milli);
    ar.put(exe.part(Q, Q), in->exe_mem_bytes);
    ar.put_or_zero(exe.part(2 * Q, Q), in->exe_gpu);
    if (has_host) {
        di.host_off = ar.put(hoff, in->host_off);
        ar.put(hn.part(0, H), in->host_nodes);
    }
    if (zoned) ar.zero(tot);
    GP_TRY(ar.check(c));
    const int T = 256;
    const int nb = (n + T - 1) / T;
    if (zoned) {
        gp_rp_zone_totals<<<nb, T, 0, st>>>(n, d_avail, d_avail + N, ni.zone, keep, ni.tz, ar.ptr(tot));
        gp_zone_priority<<<(sort->n_zones + T - 1) / T, T, 0, st>>>(sort->n_zones, sort->n_zones, ar.ptr(tot), ar.ptr(prio));
    }
    ni.avail = d_avail; ni.ff = d_ff;
    for (int d = 0; d < 3; ++d) ni.over[d] = d_over[d];
    ni.prio = ar.ptr(prio);
    ni.keep = keep; ni.n = n; ni.err = d_err;
    gp_rp_nodes<<<nb, T, 0, st>>>(ni, ar.ptr(rec));
    di.host_nodes = ar.ptr(hn);
    di.n = n; di.q = q;
    // one CTA per executor; the grid is capped at 8 CTAs per SM's worth of executors and grid-strides over the rest.  The cap
    // only sizes the grid: registers bound residency (gp_rp_decide<true>: 78 x 256 threads -> 3 CTAs per SM; <false>: 48 -> 5),
    // so the CTAs beyond that wait for a free slot
    const int blocks = (int)std::min<int64_t>(q, (int64_t)c->sm_count * 8);
    uint8_t* d_amb = ambiguous ? ar.ptr(amb) : nullptr;
    if (mf) gp_rp_decide<true><<<blocks, kRpThreads, 0, st>>>(ar.ptr(rec), di, ar.ptr(d_out), d_amb);
    else gp_rp_decide<false><<<blocks, kRpThreads, 0, st>>>(ar.ptr(rec), di, ar.ptr(d_out), d_amb);
    GP_CUDA(c, cudaGetLastError());
    ar.get(node_out, d_out);
    ar.get(ambiguous, amb);
    int err[2] = {0, 0}, gather = 0;
    ar.get(err, d_err, 2);
    if (dev) ar.get(&gather, usage.gather_err, 1);
    GP_TRY(ar.sync(c));
    GP_TRY(nt_refusal(c, gather, who));
    return stage_refusal(c, err, who);                  // refused: node_out / ambiguous hold no decision
}

extern "C" {

// rescheduleExecutor from the reservations to the node choice (SURVEY 8f row f4); see gangpack_reschedprep.cuh
gp_status gp_reschedule_from_reservations(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const gp_reschedule_scope* scope,
                                          const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous) {
    return reschedule_from_reservations(c, usage, sort, scope, in, node_out, ambiguous, "gp_reschedule_from_reservations");
}

// the same with the reservations (and optionally the overhead) from the context's resident tables
gp_status gp_reschedule_from_reservations_resident(gp_ctx* c, const gp_resident_usage* usage, const gp_sort_input* sort,
                                                   const gp_reschedule_scope* scope, const gp_reschedule* in, int32_t* node_out,
                                                   uint8_t* ambiguous) {
    return reschedule_from_reservations(c, usage, sort, scope, in, node_out, ambiguous, "gp_reschedule_from_reservations_resident");
}

}  // extern "C"

// gp_reconcile_find_nodes[_resident|_node_table].  Gathered input (usage.on_device()): node_group, creation, unschedulable
// and ready are device pointers too, kept in range by the gather, whose status word is read in the one synchronise.
static gp_status reconcile_find_nodes(gp_ctx* c, const UsageIn& usage, const gp_reconcile_nodes* nodes, const gp_apps* a,
                                      gp_reconcile_results* out, const char* who) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(check_source(c, usage, who));
    const int32_t n = usage.n_nodes();
    if (!nodes || !a || !out || nodes->n_groups < 1 || a->n_apps < 0 || (n > 0 && (!nodes->node_group || !nodes->creation)) ||
        (a->n_apps > 0 && (!a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !out->placed)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes (n_groups >= 1)");
    const int32_t q = a->n_apps, G = nodes->n_groups;
    const bool dev = usage.on_device();
    for (int32_t i = 0; i < (dev ? 0 : n); ++i)
        if (nodes->node_group[i] < 0 || nodes->node_group[i] >= G) return fail(c, GP_ERR_INVALID, who, "node_group out of range");
    GP_TRY(check_requests(c, q, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu, who));
    int64_t total = 0;
    for (int32_t i = 0; i < q; ++i) {
        const int32_t k = a->exe_count[i];
        if (k < 0) return fail(c, GP_ERR_INVALID, who, "negative exe_count");
        if (k > kMaxCount) return fail(c, GP_ERR_UNREPRESENTABLE, who, "exe_count > 2^24");
        if (a->group && (a->group[i] < 0 || a->group[i] >= G)) return fail(c, GP_ERR_INVALID, who, "instance group out of range");
        if (a->exec_out_off && a->exec_out_off[i] != total) return fail(c, GP_ERR_INVALID, who, "exec_out_off is not the prefix sum of exe_count");
        total += k;
    }
    if (a->exec_out_off && a->exec_out_off[q] != total) return fail(c, GP_ERR_INVALID, who, "exec_out_off is not the prefix sum of exe_count");
    if (total > 0 && (!out->executor_nodes || out->executor_nodes_cap < total))
        return fail(c, GP_ERR_CAPACITY, who, "executor_nodes_cap below the sum of exe_count");
    const bool want_avail = out->avail_cpu_milli || out->avail_mem_bytes || out->avail_gpu;
    if (n == 0) {                                       // every group is missing from orderedNodes
        for (int32_t i = 0; i < q; ++i) out->placed[i] = -1;
        return GP_OK;
    }
    if (q == 0 && !want_avail) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    long long *d_avail = nullptr, *d_sched = nullptr;   // usagebuf: scratch of the availability stage, charged in place below
    int* d_err = nullptr;
    GP_TRY(stage_availability(c, usage, st, &d_avail, &d_sched, &d_err));
    const size_t N = (size_t)n, Q = (size_t)q, Gs = (size_t)G, E = (size_t)total;
    Arena ar{c->callbuf, st};
    const auto grp = ar.take<int32_t>(N);
    const auto cre = ar.take<long long>(N);
    const auto fu = ar.take<uint8_t>(N), fr = ar.take<uint8_t>(N);
    const auto keys = ar.take<ReconKey>(N), sorted = ar.take<ReconKey>(N);
    const auto pos = ar.take<int32_t>(N), order = ar.take<int32_t>(N), ngrp = ar.take<int32_t>(N), noff = ar.take<int32_t>(Gs + 1),
               aoff = ar.take<int32_t>(Gs + 1);
    const auto exe = ar.take<long long>(3 * Q);
    const auto cnt = ar.take<int32_t>(Q), agrp = ar.take<int32_t>(Q);
    const auto off = ar.take<long long>(Q);
    const auto list = ar.take<int32_t>(Q);
    const auto lk = ar.take<LabelKey>(Q), lks = ar.take<LabelKey>(Q);
    const auto apos = ar.take<int32_t>(Q), apps = ar.take<int32_t>(Q), placed = ar.take<int32_t>(Q), exn = ar.take<int32_t>(E);
    const auto claim = ar.take<unsigned int>(1);
    const auto herr_p = ar.take<int>(1);
    const auto n_listed = ar.take<int32_t>(2);
    ar.reserve();
    const int32_t* d_grp = dev ? nodes->node_group : ar.put(grp, nodes->node_group);
    const long long* d_cre = dev ? (const long long*)nodes->creation : ar.put(cre, nodes->creation);
    const uint8_t* d_fu = dev ? nodes->unschedulable : ar.put(fu, nodes->unschedulable);
    const uint8_t* d_fr = dev ? nodes->ready : ar.put(fr, nodes->ready);
    ar.fill(claim, n_listed, 0);                        // claim counter, error word, listed drivers
    GP_TRY(ar.check(c));
    if (!c->recon_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<ReconKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(ReconKey))));
        c->recon_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    gp_rc_node_keys<<<nb, T, 0, st>>>(n, G, d_grp, d_cre, d_fu, d_fr, ar.ptr(keys), ar.ptr(ngrp));
    gp_sort_tiles<ReconKey><<<(n + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(ReconKey), st>>>(n, nullptr, ar.ptr(keys), ar.ptr(sorted));
    gp_rank_by_search<ReconKey><<<nb, T, 0, st>>>(n, nullptr, ar.ptr(keys), ar.ptr(sorted), ar.ptr(pos));
    gp_scatter_order<<<nb, T, 0, st>>>(n, ar.ptr(pos), ar.ptr(order));
    if (q > 0) {
        // exe cpu, mem, gpu columns, counts, groups and offsets
        ar.put(exe.part(0, Q), a->exe_cpu_milli);
        ar.put(exe.part(Q, Q), a->exe_mem_bytes);
        ar.put_or_zero(exe.part(2 * Q, Q), a->exe_gpu);
        ar.put(cnt, a->exe_count);
        ar.put_or_zero(agrp, a->group);
        if (a->exec_out_off) ar.put(off, a->exec_out_off);
        else {
            std::vector<int64_t>& h = c->host_off;
            h.resize(Q);
            int64_t run = 0;
            for (int32_t i = 0; i < q; ++i) { h[i] = run; run += a->exe_count[i]; }
            ar.put(off, h.data());
        }
        GP_TRY(ar.check(c));
        // the stale drivers partitioned by group, call order kept inside each group
        const int qb = (q + T - 1) / T;
        gp_rc_app_list<<<qb, T, 0, st>>>(q, ar.ptr(list), ar.ptr(n_listed));
        launch_label_resort(q, ar.ptr(n_listed), ar.ptr(list), ar.ptr(agrp), ar.ptr(lk), ar.ptr(lks), ar.ptr(apos), ar.ptr(apps), st);
    }
    gp_rc_offsets<<<(unsigned)((Gs + T) / T), T, 0, st>>>(G, n, ar.ptr(order), ar.ptr(ngrp), q, ar.ptr(apps), ar.ptr(agrp), ar.ptr(noff),
                                                          ar.ptr(aoff));
    if (q > 0) {
        RcLoopIn li{};
        li.avail = d_avail; li.order = ar.ptr(order); li.noff = ar.ptr(noff);
        li.apps = ar.ptr(apps); li.aoff = ar.ptr(aoff);
        li.exe = ar.ptr(exe); li.count = ar.ptr(cnt); li.out_off = ar.ptr(off);
        li.placed = ar.ptr(placed); li.exec_nodes = ar.ptr(exn);
        li.claim = ar.ptr(claim); li.err = ar.ptr(herr_p);
        li.n = n; li.q = q; li.n_groups = G;
        // one CTA per instance group; CTAs that find no group left return at once
        const int blocks = (int)std::min<int64_t>(G, (int64_t)c->sm_count * 8);
        gp_rc_loop<<<blocks, kRcThreads, 0, st>>>(li);
    }
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    if (q > 0) {
        ar.get(out->placed, placed);
        ar.get(out->executor_nodes, exn);
        ar.get(&herr, herr_p);
    }
    int64_t* outs[3] = {out->avail_cpu_milli, out->avail_mem_bytes, out->avail_gpu};
    for (int d = 0; d < 3; ++d) ar.get(outs[d], d_avail + N * (size_t)d, N);
    int uerr[2] = {0, 0}, gather = 0;
    ar.get(uerr, d_err, 2);
    if (dev) ar.get(&gather, usage.gather_err, 1);
    GP_TRY(ar.sync(c));
    GP_TRY(nt_refusal(c, gather, who));
    GP_TRY(stage_refusal(c, uerr, who));
    return refuse(c, herr, kRcRefusals, who);
}

extern "C" {

// the failover reconciler's findNodes loop for a batch of stale drivers (EXT/failover.go:43-82, 286-436); see
// gangpack_reconcile.cuh and DESIGN §2.3
gp_status gp_reconcile_find_nodes(gp_ctx* c, const gp_usage_input* usage, const gp_reconcile_nodes* nodes, const gp_apps* a,
                                  gp_reconcile_results* out) {
    return reconcile_find_nodes(c, usage, nodes, a, out, "gp_reconcile_find_nodes");
}

// the same with the reservations (and optionally the overhead) from the context's resident tables
gp_status gp_reconcile_find_nodes_resident(gp_ctx* c, const gp_resident_usage* usage, const gp_reconcile_nodes* nodes, const gp_apps* a,
                                           gp_reconcile_results* out) {
    return reconcile_find_nodes(c, usage, nodes, a, out, "gp_reconcile_find_nodes_resident");
}

}  // extern "C"

// ---- the *_node_table forms: nt_gather fills the columns on the device, then the *_resident entry's own path runs ----

extern "C" {

gp_status gp_prepare_cluster_groups_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, const int32_t* instance_group,
                                               int32_t n_instance_groups, gp_instance_group_orders* out) {
    static const char* who = "gp_prepare_cluster_groups_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, instance_group, n_instance_groups, true, who, &g));
    GP_TRY(check_instance_groups(c, UsageIn(&g.usage), &g.sort, instance_group, n_instance_groups, who));
    GP_TRY(prepare_cluster_groups(c, UsageIn(&g.usage, g.err), &g.sort, g.ig, n_instance_groups, out, who));
    return nt_outputs(c, nodes, g);
}

gp_status gp_prepare_cluster_zones_groups_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, const int32_t* instance_group,
                                                     int32_t n_instance_groups, gp_instance_group_layout* layout) {
    static const char* who = "gp_prepare_cluster_zones_groups_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, instance_group, n_instance_groups, true, who, &g));
    GP_TRY(check_instance_groups(c, UsageIn(&g.usage), &g.sort, instance_group, n_instance_groups, who));
    GP_TRY(prepare_cluster_zones_groups(c, UsageIn(&g.usage, g.err), &g.sort, g.ig, n_instance_groups, layout, who));
    return nt_outputs(c, nodes, g);
}

gp_status gp_reschedule_from_reservations_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, const gp_reschedule_scope* scope,
                                                     const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous) {
    static const char* who = "gp_reschedule_from_reservations_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, nullptr, 1, false, who, &g));
    GP_TRY(reschedule_from_reservations(c, UsageIn(&g.usage, g.err), &g.sort, scope, in, node_out, ambiguous, who));
    return nt_outputs(c, nodes, g);
}

// the failover reconciler: the gather adds creation and the reconciler's instance groups, then gp_reconcile_find_nodes_resident's
// path runs on them
gp_status gp_reconcile_find_nodes_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, int32_t n_groups, int32_t instance_group_missing,
                                             const gp_apps* a, gp_reconcile_results* out) {
    static const char* who = "gp_reconcile_find_nodes_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    NtGathered g{};
    const NtReconcile rc{instance_group_missing};
    GP_TRY(nt_gather(c, nodes, nullptr, n_groups, true, who, &g, &rc));
    gp_reconcile_nodes rn{};
    rn.n_groups = n_groups;
    rn.node_group = g.ig;
    rn.creation = (const int64_t*)g.creation;
    rn.unschedulable = g.sort.unschedulable;
    rn.ready = g.sort.ready;
    GP_TRY(reconcile_find_nodes(c, UsageIn(&g.usage, g.err), &rn, a, out, who));
    return nt_outputs(c, nodes, g);
}

}  // extern "C"
