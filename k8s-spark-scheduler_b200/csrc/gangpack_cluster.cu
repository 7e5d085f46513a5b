// gangpack_cluster.cu -- the entry points driven by the reservations: node priority orders (gp_potential_nodes),
// availability (gp_build_*availability), the prepared snapshots (gp_prepare_cluster, gp_prepare_cluster_zones), executor
// reschedule (gp_reschedule_executors, gp_reschedule_from_reservations) and the failover reconciler (gp_reconcile_find_nodes),
// with the input checks and device staging they share.
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

// offsets of the single instance group from the device-resident candidate counts
__global__ void gp_offsets_from_counts(const int32_t* __restrict__ counts, int32_t* __restrict__ exec_off, int32_t* __restrict__ drv_off) {
    if (threadIdx.x == 0) { drv_off[0] = 0; drv_off[1] = counts[0]; exec_off[0] = 0; exec_off[1] = counts[1]; }
}

// Host checks shared by the entries below; `who` (the entry's name) prefixes every message.  The shape of a gp_usage_input:
// sizes non-negative, the allocatable columns for nodes, the reservation columns for rows, fewer than 2^31 rows (the bound
// the exact usage sums rest on).  The quantities themselves are checked where they are read, on the device (usage_refusal).
static gp_status check_usage(gp_ctx* c, const gp_usage_input* in, const char* who) {
    if (!in || in->n_nodes < 0 || in->n_reservations < 0 || in->n_reservations > 0x7fffffffLL ||
        (in->n_nodes > 0 && (!in->alloc_cpu_milli || !in->alloc_mem_bytes)) ||
        (in->n_reservations > 0 && (!in->res_node || !in->res_cpu_milli || !in->res_mem_bytes)))
        return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or bad sizes");
    return GP_OK;
}

// The status word of the availability stage (kFeErr* bits), read back by the entry: the refusal it stands for.
static gp_status usage_refusal(gp_ctx* c, int err, const char* who) {
    if (err & kFeErrInput)
        return fail(c, GP_ERR_UNREPRESENTABLE, std::string(who) + ": |allocatable|, |overhead| or |reservation| >= 2^61");
    if (err & kFeErrResult)
        return fail(c, GP_ERR_UNREPRESENTABLE, std::string(who) + ": a node's reservation sum or availability lies outside the exact-int64 domain (|v| >= 2^61)");
    return GP_OK;
}

// The two id arrays of a gp_sort_input the kernels index with: zone ids in range, name ranks a permutation of 0..n-1 (a rank
// given twice would leave a position of the order unwritten).
static gp_status check_sort_ids(gp_ctx* c, const gp_sort_input* in, const char* who) {
    const int32_t n = in->n_nodes;
    if (in->zone_id) for (int32_t i = 0; i < n; ++i)
        if (in->zone_id[i] < 0 || in->zone_id[i] >= in->n_zones) return fail(c, GP_ERR_INVALID, std::string(who) + ": zone_id out of range");
    if (in->name_rank) {
        std::vector<uint8_t>& seen = c->v_seen_e;       // host scratch of the order checks
        seen.assign((size_t)n, 0);
        for (int32_t i = 0; i < n; ++i) {
            const int32_t r = in->name_rank[i];
            if (r < 0 || r >= n) return fail(c, GP_ERR_INVALID, std::string(who) + ": name_rank out of range");
            if (seen[r]) return fail(c, GP_ERR_INVALID, std::string(who) + ": name_rank is not a permutation (a rank is given twice)");
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
            if (x < 0) return fail(c, GP_ERR_INVALID, std::string(who) + ": negative resource request");
            if (x >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, std::string(who) + ": quantity >= 2^61");
        }
    }
    return GP_OK;
}

// The host_off / host_nodes CSR of a gp_reschedule (host_off given): monotone from 0, node indices below n_nodes.
// *hosted = host_off[n_execs].
static gp_status check_hosting(gp_ctx* c, const gp_reschedule* in, int32_t n_nodes, int64_t* hosted, const char* who) {
    const std::string w(who);
    if (in->host_off[0] != 0) return fail(c, GP_ERR_INVALID, w + ": host_off must start at 0");
    for (int32_t i = 0; i < in->n_execs; ++i)
        if (in->host_off[i + 1] < in->host_off[i]) return fail(c, GP_ERR_INVALID, w + ": host_off not monotone");
    *hosted = in->host_off[in->n_execs];
    if (*hosted > 0 && !in->host_nodes) return fail(c, GP_ERR_INVALID, w + ": host_nodes missing");
    for (int64_t t = 0; t < *hosted; ++t)
        if (in->host_nodes[t] < 0 || in->host_nodes[t] >= n_nodes) return fail(c, GP_ERR_INVALID, w + ": host_nodes index out of range");
    return GP_OK;
}

// f2 stage: uploads the inputs, leaves avail[3][N] / sched[3][N] and the stage's status word (*d_err: kFeErr* bits, for
// usage_refusal once the stream has been synchronised) on the device (usagebuf).
// d_over (optional, [3]): the uploaded overhead columns, NULL where the caller gave none.
static gp_status stage_availability(gp_ctx* c, const gp_usage_input* in, cudaStream_t st, long long** d_avail, long long** d_sched, int** d_err,
                                    long long** d_resched = nullptr, const long long** d_over = nullptr) {
    const int32_t n = in->n_nodes;
    const size_t N = (size_t)n, R = (size_t)in->n_reservations;
    Arena ar{c->usagebuf};
    const size_t o_alloc = ar.take(24 * N), o_over = ar.take(24 * N), o_usage = ar.take(48 * N + 4 * N + 4), o_avail = ar.take(24 * N),
                 o_sched = ar.take(24 * N), o_resched = ar.take(24 * N), o_rn = ar.take(4 * R), o_rc = ar.take(8 * R), o_rm = ar.take(8 * R),
                 o_rg = ar.take(8 * R);
    const size_t o_has = o_usage + 48 * N, o_err = o_has + 4 * N;      // zeroed together with the usage sums
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, ar.upload(o_alloc, in->alloc_cpu_milli, 8 * N, st));
    GP_CUDA(c, ar.upload(o_alloc + 8 * N, in->alloc_mem_bytes, 8 * N, st));
    if (in->alloc_gpu) GP_CUDA(c, ar.upload(o_alloc + 16 * N, in->alloc_gpu, 8 * N, st));
    if (in->overhead_cpu_milli) GP_CUDA(c, ar.upload(o_over, in->overhead_cpu_milli, 8 * N, st));
    if (in->overhead_mem_bytes) GP_CUDA(c, ar.upload(o_over + 8 * N, in->overhead_mem_bytes, 8 * N, st));
    if (in->overhead_gpu) GP_CUDA(c, ar.upload(o_over + 16 * N, in->overhead_gpu, 8 * N, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_usage, 0, 52 * N + 4, st));
    const int T = 256;
    int* err = (int*)(b + o_err);
    if (R) {
        GP_CUDA(c, ar.upload(o_rn, in->res_node, 4 * R, st));
        GP_CUDA(c, ar.upload(o_rc, in->res_cpu_milli, 8 * R, st));
        GP_CUDA(c, ar.upload(o_rm, in->res_mem_bytes, 8 * R, st));
        if (in->res_gpu) GP_CUDA(c, ar.upload(o_rg, in->res_gpu, 8 * R, st));
        gp_usage_scatter<<<(unsigned)((R + T - 1) / T), T, 0, st>>>((long long)R, (const int32_t*)(b + o_rn), (const long long*)(b + o_rc),
                                                                   (const long long*)(b + o_rm), in->res_gpu ? (const long long*)(b + o_rg) : nullptr,
                                                                   n, (unsigned long long*)(b + o_usage), d_resched ? (unsigned int*)(b + o_has) : nullptr, err);
    }
    const long long* al = (const long long*)(b + o_alloc);
    const long long* ov = (const long long*)(b + o_over);
    gp_availability<<<(n + T - 1) / T, T, 0, st>>>(n, al, al + N, in->alloc_gpu ? al + 2 * N : nullptr, in->overhead_cpu_milli ? ov : nullptr,
                                                   in->overhead_mem_bytes ? ov + N : nullptr, in->overhead_gpu ? ov + 2 * N : nullptr,
                                                   (const unsigned long long*)(b + o_usage), (long long*)(b + o_avail), (long long*)(b + o_sched), err,
                                                   (const unsigned int*)(b + o_has), d_resched ? (long long*)(b + o_resched) : nullptr);
    if (d_resched) *d_resched = (long long*)(b + o_resched);
    if (d_over) {
        d_over[0] = in->overhead_cpu_milli ? ov : nullptr;
        d_over[1] = in->overhead_mem_bytes ? ov + N : nullptr;
        d_over[2] = in->overhead_gpu ? ov + 2 * N : nullptr;
    }
    GP_CUDA(c, cudaGetLastError());
    *d_avail = (long long*)(b + o_avail);
    *d_sched = (long long*)(b + o_sched);
    *d_err = err;
    return GP_OK;
}

struct SortStage { const int32_t* drv; const int32_t* exe; const int32_t* counts; const int32_t* zone; };

// Stable re-sort of list[0..*cnt) by rank[node] (-1 last): out[k] = the k-th node in (rank, position) order.  The label
// re-sort of PotentialNodes, and the zone partition of gp_prepare_cluster_zones.
static void launch_label_resort(int32_t n, const int32_t* cnt, const int32_t* list, const int32_t* rank, LabelKey* lk, LabelKey* lks,
                                int32_t* pos, int32_t* out, cudaStream_t st) {
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    gp_label_keys<<<nb, T, 0, st>>>(cnt, list, rank, lk);
    gp_sort_tiles<LabelKey><<<ntile, kSortThreads, kSortTile * sizeof(LabelKey), st>>>(n, cnt, lk, lks);
    gp_rank_by_search<LabelKey><<<nb, T, 0, st>>>(n, cnt, lk, lks, pos);
    gp_label_scatter<<<nb, T, 0, st>>>(cnt, list, pos, out);
}

// f1 stage: d_cpu / d_mem / d_gpu are device arrays (NULL: uploaded from `in`; gpu optional); leaves the two orders,
// counts[3] = {#driver candidates, #executor candidates, #undefined ties} and the zone ids (NULL: one zone) on the device.
// The caller has run check_sort_ids.
static gp_status stage_sort(gp_ctx* c, const gp_sort_input* in, const long long* d_cpu, const long long* d_mem, const long long* d_gpu,
                            cudaStream_t st, SortStage* out) {
    const int32_t n = in->n_nodes;
    // one scratch block
    const size_t N = (size_t)n, Z = (size_t)in->n_zones;
    Arena ar{c->sortbuf};
    const size_t o_cpu = ar.take(8 * N), o_mem = ar.take(8 * N), o_gpu = ar.take(8 * N), o_keys = ar.take(sizeof(SortKey) * N),
                 o_sorted = ar.take(sizeof(SortKey) * N), o_tot = ar.take(8 * kZoneTotWords * Z), o_zone = ar.take(4 * N), o_nr = ar.take(4 * N),
                 o_prio = ar.take(4 * Z), o_pos = ar.take(4 * N), o_order = ar.take(4 * N), o_drv = ar.take(4 * N), o_exe = ar.take(4 * N),
                 o_drv2 = ar.take(4 * N), o_exe2 = ar.take(4 * N), o_lrd = ar.take(4 * N), o_lre = ar.take(4 * N),
                 o_lk = ar.take(sizeof(LabelKey) * N), o_lks = ar.take(sizeof(LabelKey) * N), o_cnt = ar.take(16),
                 o_fc = ar.take(N), o_fu = ar.take(N), o_fr = ar.take(N);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    if (!d_cpu) { GP_CUDA(c, ar.upload(o_cpu, in->avail_cpu_milli, 8 * N, st)); d_cpu = (const long long*)(b + o_cpu); }
    if (!d_mem) { GP_CUDA(c, ar.upload(o_mem, in->avail_mem_bytes, 8 * N, st)); d_mem = (const long long*)(b + o_mem); }
    if (!d_gpu && in->avail_gpu) { GP_CUDA(c, ar.upload(o_gpu, in->avail_gpu, 8 * N, st)); d_gpu = (const long long*)(b + o_gpu); }
    const bool zoned = in->zone_id != nullptr && in->n_zones > 1;       // one zone: priority 0 for every node, nothing to total
    if (zoned) GP_CUDA(c, ar.upload(o_zone, in->zone_id, 4 * N, st));
    if (in->name_rank) GP_CUDA(c, ar.upload(o_nr, in->name_rank, 4 * N, st));
    if (in->is_driver_candidate) GP_CUDA(c, ar.upload(o_fc, in->is_driver_candidate, N, st));
    if (in->unschedulable) GP_CUDA(c, ar.upload(o_fu, in->unschedulable, N, st));
    if (in->ready) GP_CUDA(c, ar.upload(o_fr, in->ready, N, st));
    if (in->driver_label_rank) GP_CUDA(c, ar.upload(o_lrd, in->driver_label_rank, 4 * N, st));
    if (in->executor_label_rank) GP_CUDA(c, ar.upload(o_lre, in->executor_label_rank, 4 * N, st));
    if (zoned) GP_CUDA(c, cudaMemsetAsync(b + o_tot, 0, 8 * kZoneTotWords * Z, st));
    if (!c->sort_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<SortKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(SortKey))));
        c->sort_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    SortKey* keys = (SortKey*)(b + o_keys);
    SortKey* sorted = (SortKey*)(b + o_sorted);
    int32_t* pos = (int32_t*)(b + o_pos);
    if (zoned) {
        gp_zone_totals<<<nb, T, 0, st>>>(n, d_cpu, d_mem, (const int32_t*)(b + o_zone), (unsigned long long*)(b + o_tot));
        gp_zone_priority<<<(in->n_zones + T - 1) / T, T, 0, st>>>(in->n_zones, (const unsigned long long*)(b + o_tot), (int32_t*)(b + o_prio));
    }
    gp_make_keys<<<nb, T, 0, st>>>(n, d_cpu, d_mem, zoned ? (const int32_t*)(b + o_zone) : nullptr, (const int32_t*)(b + o_prio),
                                   in->name_rank ? (const int32_t*)(b + o_nr) : nullptr, keys);
    gp_sort_tiles<SortKey><<<ntile, kSortThreads, kSortTile * sizeof(SortKey), st>>>(n, nullptr, keys, sorted);
    gp_rank_by_search<SortKey><<<nb, T, 0, st>>>(n, nullptr, keys, sorted, pos);
    gp_scatter_order<<<nb, T, 0, st>>>(n, pos, (int32_t*)(b + o_order));
    gp_split_candidates<<<1, 1024, 0, st>>>(n, (const int32_t*)(b + o_order), in->is_driver_candidate ? (const uint8_t*)(b + o_fc) : nullptr,
                                           in->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr, in->ready ? (const uint8_t*)(b + o_fr) : nullptr,
                                           keys, d_gpu, (int32_t*)(b + o_drv), (int32_t*)(b + o_exe), (int32_t*)(b + o_cnt));
    out->drv = (const int32_t*)(b + o_drv);
    out->exe = (const int32_t*)(b + o_exe);
    out->counts = (const int32_t*)(b + o_cnt);
    out->zone = zoned ? (const int32_t*)(b + o_zone) : nullptr;
    auto label_sort = [&](const int32_t* cnt, const int32_t* list, size_t o_rank, size_t o_out) {
        launch_label_resort(n, cnt, list, (const int32_t*)(b + o_rank), (LabelKey*)(b + o_lk), (LabelKey*)(b + o_lks), pos,
                            (int32_t*)(b + o_out), st);
        return (const int32_t*)(b + o_out);
    };
    if (in->driver_label_rank) out->drv = label_sort(out->counts, out->drv, o_lrd, o_drv2);
    if (in->executor_label_rank) out->exe = label_sort(out->counts + 1, out->exe, o_lre, o_exe2);
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// gp_prepare_cluster and gp_prepare_cluster_zones up to their layout step: the checks both make, then reservations ->
// availability (d_avail / d_sched: [3][n_nodes]) -> priority orders on the context's stream.  Synchronises once for the
// availability stage's status word: a refusal returns before anything of the context's snapshot has been replaced.
static gp_status prepare_orders(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const char* who,
                                long long** d_avail, long long** d_sched, SortStage* so) {
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!sort || usage->n_nodes != sort->n_nodes || sort->n_zones < 1)
        return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or mismatched sizes");
    if (usage->n_nodes == 0) return fail(c, GP_ERR_INVALID, std::string(who) + ": empty node table");
    if ((s = check_sort_ids(c, sort, who)) != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    int* d_err = nullptr;
    if ((s = stage_availability(c, usage, c->stream, d_avail, d_sched, &d_err)) != GP_OK) return s;
    const size_t N = (size_t)usage->n_nodes;
    if ((s = stage_sort(c, sort, *d_avail, *d_avail + N, *d_avail + 2 * N, c->stream, so)) != GP_OK) return s;
    int err = 0;
    GP_CUDA(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, c->stream));
    GP_CUDA(c, cudaStreamSynchronize(c->stream));
    return usage_refusal(c, err, who);
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
    if ((s = usage_refusal(c, err, who)) != GP_OK) return s;           // the outputs are left as they were
    const size_t N = (size_t)n;
    const long long* src[2] = {first_fit ? d_ff : d_avail, d_sched};
    for (int k = 0; k < 6; ++k)
        if (outs[k]) GP_CUDA(c, cudaMemcpyAsync(outs[k], src[k / 3] + N * (size_t)(k % 3), 8 * N, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

extern "C" {

gp_status gp_potential_nodes(gp_ctx* c, const gp_sort_input* in, int32_t* driver_order, int32_t* n_driver,
                             int32_t* executor_order, int32_t* n_executor) {
    if (!c) return GP_ERR_INVALID;
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
    s = stage_sort(c, in, nullptr, nullptr, nullptr, st, &so);
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
    if (!c) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, sched_cpu, sched_mem, sched_gpu};
    return availability_out(c, in, false, outs, "gp_build_availability");
}

// availableResources of rescheduleExecutor's first-fit branch: the availability to upload before gp_reschedule_executors(min_frag = 0)
gp_status gp_build_reschedule_availability(gp_ctx* c, const gp_usage_input* in, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu) {
    if (!c) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, nullptr, nullptr, nullptr};
    return availability_out(c, in, true, outs, "gp_build_reschedule_availability");
}

// reservations -> availability -> priority orders -> slot layout, without leaving the device
gp_status gp_prepare_cluster(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, int32_t* n_driver, int32_t* n_executor) {
    if (!c) return GP_ERR_INVALID;
    if (n_driver) *n_driver = 0;
    if (n_executor) *n_executor = 0;
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    gp_status s = prepare_orders(c, usage, sort, "gp_prepare_cluster", &d_avail, &d_sched, &so);
    if (s != GP_OK) return s;
    cudaStream_t st = c->stream;
    GP_CUDA(c, c->exec_off.reserve(8)); GP_CUDA(c, c->drv_off.reserve(8));
    gp_offsets_from_counts<<<1, 32, 0, st>>>(so.counts, c->exec_off.as<int32_t>(), c->drv_off.as<int32_t>());
    gp_nodes dn{};
    dn.n_nodes = usage->n_nodes;
    dn.n_groups = 1;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = so.exe;
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = so.drv;
    int32_t counts[3] = {0, 0, 0};
    s = prepare_snapshot(c, &dn, d_avail, d_sched, so, counts);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaStreamSynchronize(st));
    c->n_drv = counts[0]; c->n_exec = counts[1];
    c->have_eff_sched = true;           // SchedulableResources for gp_packing_efficiency (the zone entry points still want gp_set_schedulable)
    if (sort->undefined_ties) *sort->undefined_ties = counts[2];
    if (n_driver) *n_driver = counts[0];
    if (n_executor) *n_executor = counts[1];
    return GP_OK;
}

// reservations -> availability -> priority orders -> zone-grouped slot layout, without leaving the device
gp_status gp_prepare_cluster_zones(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, gp_zone_layout* layout) {
    if (!c) return GP_ERR_INVALID;
    if (!layout) return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: missing arrays or mismatched sizes");
    const int32_t kind = layout->kind;
    if (kind != GP_LAYOUT_SINGLE_AZ && kind != GP_LAYOUT_AZ_AWARE)
        return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: layout->kind must be GP_LAYOUT_SINGLE_AZ or GP_LAYOUT_AZ_AWARE");
    if (sort && sort->n_zones == 0x7fffffff) return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: n_zones too large");
    layout->n_zones = 0; layout->n_groups = 0; layout->n_driver = 0; layout->n_executor = 0;
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    gp_status s = prepare_orders(c, usage, sort, "gp_prepare_cluster_zones", &d_avail, &d_sched, &so);
    if (s != GP_OK) return s;
    cudaStream_t st = c->stream;
    c->zone_kind = -1;                                  // the held orders are overwritten below
    const int32_t n = usage->n_nodes;
    const size_t N = (size_t)n;
    // g_bound = sort->n_zones + 1 groups bound every layout; the slots are laid out for that many (the groups past the
    // last one are empty) so that the group count can stay on the device until the one synchronise below
    const size_t Zs = (size_t)sort->n_zones;
    const int32_t g_bound = sort->n_zones + 1;
    Arena ar{c->zoneprep};
    const size_t o_udrv = ar.take(4 * N), o_uexe = ar.take(4 * N), o_first = ar.take(4 * Zs), o_has = ar.take(Zs), o_zg = ar.take(4 * Zs),
                 o_zog = ar.take(4 * (Zs + 1)), o_rank = ar.take(4 * N), o_lk = ar.take(sizeof(LabelKey) * N), o_lks = ar.take(sizeof(LabelKey) * N),
                 o_pos = ar.take(4 * N), o_info = ar.take(4 * kZiWords);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    int32_t* udrv = (int32_t*)(b + o_udrv);
    int32_t* uexe = (int32_t*)(b + o_uexe);
    int32_t* info = (int32_t*)(b + o_info);
    int32_t* rank = (int32_t*)(b + o_rank);
    // the undivided orders outlive the sort's scratch, which the next gp_potential_nodes / gp_prepare_cluster reuses
    GP_CUDA(c, cudaMemcpyAsync(udrv, so.drv, 4 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(uexe, so.exe, 4 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_first, 0x7f, 4 * Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_has, 0, Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_zg, 0xff, 4 * Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_zog, 0xff, 4 * (Zs + 1), st));
    GP_CUDA(c, cudaMemsetAsync(info, 0, 4 * kZiWords, st));
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int32_t az = kind == GP_LAYOUT_AZ_AWARE ? 1 : 0;
    gp_zone_mark<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, (int32_t*)(b + o_first), (uint8_t*)(b + o_has));
    gp_zone_candidates<<<1, 1024, 0, st>>>(so.counts, udrv, so.zone, (const int32_t*)(b + o_first), (const uint8_t*)(b + o_has),
                                           (int32_t*)(b + o_zg), (int32_t*)(b + o_zog), info);
    gp_group_rank<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, (const int32_t*)(b + o_zg), az, info, rank);
    GP_CUDA(c, cudaGetLastError());
    // the grouped orders and their offsets
    GP_CUDA(c, c->exec_order.reserve(4 * (N + 1))); GP_CUDA(c, c->drv_order.reserve(4 * (N + 1)));
    GP_CUDA(c, c->exec_off.reserve(4 * ((size_t)g_bound + 1))); GP_CUDA(c, c->drv_off.reserve(4 * ((size_t)g_bound + 1)));
    LabelKey* lk = (LabelKey*)(b + o_lk);
    LabelKey* lks = (LabelKey*)(b + o_lks);
    int32_t* pos = (int32_t*)(b + o_pos);
    launch_label_resort(n, so.counts, udrv, rank, lk, lks, pos, c->drv_order.as<int32_t>(), st);
    launch_label_resort(n, so.counts + 1, uexe, rank, lk, lks, pos, c->exec_order.as<int32_t>(), st);
    gp_group_offsets<<<(unsigned)((g_bound + T) / T), T, 0, st>>>(g_bound, so.counts, c->drv_order.as<int32_t>(), c->exec_order.as<int32_t>(),
                                                                  rank, az, c->exec_off.as<int32_t>(), c->drv_off.as<int32_t>(), info);
    GP_CUDA(c, cudaGetLastError());
    gp_nodes dn{};
    dn.n_nodes = n;
    dn.n_groups = g_bound;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = c->exec_order.as<int32_t>();
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = c->drv_order.as<int32_t>();
    int32_t counts[3] = {0, 0, 0}, hinfo[kZiWords] = {};
    s = prepare_snapshot(c, &dn, d_avail, d_sched, so, counts);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(hinfo, info, sizeof(hinfo), cudaMemcpyDeviceToHost, st));
    if (layout->zone_of_group) GP_CUDA(c, cudaMemcpyAsync(layout->zone_of_group, b + o_zog, 4 * (Zs + 1), cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    c->n_groups = hinfo[kZiGroups]; c->n_exec = hinfo[kZiExec]; c->n_drv = hinfo[kZiDrv];
    c->have_sched = true;
    c->have_eff_sched = true;
    c->zone_orders = gp_az_orders{hinfo[kZiZones], counts[1], uexe, counts[0], udrv};
    c->zone_kind = kind;
    if (sort->undefined_ties) *sort->undefined_ties = counts[2];
    layout->n_zones = hinfo[kZiZones]; layout->n_groups = hinfo[kZiGroups];
    layout->n_driver = counts[0]; layout->n_executor = counts[1];
    // the grouped layout itself only when asked: its sizes are known now
    const size_t ob = 4 * (size_t)(hinfo[kZiGroups] + 1);
    if (layout->exec_off) GP_CUDA(c, cudaMemcpyAsync(layout->exec_off, c->exec_off.p, ob, cudaMemcpyDeviceToHost, st));
    if (layout->drv_off) GP_CUDA(c, cudaMemcpyAsync(layout->drv_off, c->drv_off.p, ob, cudaMemcpyDeviceToHost, st));
    if (layout->exec_order && c->n_exec) GP_CUDA(c, cudaMemcpyAsync(layout->exec_order, c->exec_order.p, 4 * (size_t)c->n_exec, cudaMemcpyDeviceToHost, st));
    if (layout->drv_order && c->n_drv) GP_CUDA(c, cudaMemcpyAsync(layout->drv_order, c->drv_order.p, 4 * (size_t)c->n_drv, cudaMemcpyDeviceToHost, st));
    if (layout->exec_off || layout->drv_off || layout->exec_order || layout->drv_order) GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

// rescheduleExecutor's node choice for a batch of executors (SURVEY 8f row f4); see gangpack_resched.cuh
gp_status gp_reschedule_executors(gp_ctx* c, const gp_reschedule* in, int32_t* node_out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_reschedule_executors: gp_set_snapshot first");
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
    Arena ar{c->reschedbuf};
    const size_t o_exe = ar.take(8 * 3 * Q), o_res = ar.take(8 * 3 * N), o_hoff = ar.take(8 * (Q + 1)), o_grp = ar.take(4 * Q),
                 o_hn = ar.take(4 * (H + 1)), o_out = ar.take(4 * Q), o_err = ar.take(8);
    GP_CUDA(c, ar.reserve());
    char* base = ar.base();
    int64_t* d_exe = reinterpret_cast<int64_t*>(base + o_exe);
    int64_t* d_res = reinterpret_cast<int64_t*>(base + o_res);
    int64_t* d_hoff = reinterpret_cast<int64_t*>(base + o_hoff);
    int32_t* d_grp = reinterpret_cast<int32_t*>(base + o_grp);
    int32_t* d_hn = reinterpret_cast<int32_t*>(base + o_hn);
    int32_t* d_out = reinterpret_cast<int32_t*>(base + o_out);
    int* d_err = reinterpret_cast<int*>(base + o_err);
    GP_CUDA(c, cudaMemsetAsync(d_err, 0, 8, st));
    GP_CUDA(c, cudaMemcpyAsync(d_exe, in->exe_cpu_milli, 8 * Q, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(d_exe + Q, in->exe_mem_bytes, 8 * Q, cudaMemcpyHostToDevice, st));
    if (in->exe_gpu) GP_CUDA(c, cudaMemcpyAsync(d_exe + 2 * Q, in->exe_gpu, 8 * Q, cudaMemcpyHostToDevice, st));
    if (in->group) GP_CUDA(c, cudaMemcpyAsync(d_grp, in->group, 4 * Q, cudaMemcpyHostToDevice, st));
    if (has_res && N) {
        GP_CUDA(c, cudaMemcpyAsync(d_res, in->reserved_cpu_milli, 8 * N, cudaMemcpyHostToDevice, st));
        GP_CUDA(c, cudaMemcpyAsync(d_res + N, in->reserved_mem_bytes, 8 * N, cudaMemcpyHostToDevice, st));
        if (in->reserved_gpu) GP_CUDA(c, cudaMemcpyAsync(d_res + 2 * N, in->reserved_gpu, 8 * N, cudaMemcpyHostToDevice, st));
    }
    if (has_host) {
        GP_CUDA(c, cudaMemcpyAsync(d_hoff, in->host_off, 8 * (Q + 1), cudaMemcpyHostToDevice, st));
        if (H) GP_CUDA(c, cudaMemcpyAsync(d_hn, in->host_nodes, 4 * H, cudaMemcpyHostToDevice, st));
    }
    ReschedIn ri{};
    ri.exe_cpu = d_exe; ri.exe_mem = d_exe + Q; ri.exe_gpu = in->exe_gpu ? d_exe + 2 * Q : nullptr;
    ri.group = in->group ? d_grp : nullptr;
    ri.res_cpu = has_res ? d_res : nullptr; ri.res_mem = has_res ? d_res + N : nullptr;
    ri.res_gpu = (has_res && in->reserved_gpu) ? d_res + 2 * N : nullptr;
    ri.host_off = has_host ? d_hoff : nullptr; ri.host_nodes = d_hn;
    ri.node_slot = c->node_slot.as<int32_t>();
    ri.n_execs = q;
    const Snapshot s = make_snapshot(c);
    const int T = 256;
    int64_t blocks = ((int64_t)q * 32 + T - 1) / T;
    const int64_t max_blocks = (int64_t)c->sm_count * 8;
    if (blocks > max_blocks) blocks = max_blocks;
    if (mf) gp_reschedule_kernel<true><<<(int)blocks, T, 0, st>>>(s, ri, d_out, d_err);
    else gp_reschedule_kernel<false><<<(int)blocks, T, 0, st>>>(s, ri, d_out, d_err);
    GP_CUDA(c, cudaGetLastError());
    int err = 0;
    GP_CUDA(c, cudaMemcpyAsync(node_out, d_out, 4 * Q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (err) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: instance group out of range");
    return GP_OK;
}

// rescheduleExecutor from the reservations to the node choice (SURVEY 8f row f4); see gangpack_reschedprep.cuh
gp_status gp_reschedule_from_reservations(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const gp_reschedule_scope* scope,
                                          const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_reschedule_from_reservations";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!sort || !in || usage->n_nodes != sort->n_nodes || sort->n_zones < 1 ||
        in->n_execs < 0 || (in->n_execs > 0 && (!in->exe_cpu_milli || !in->exe_mem_bytes || !node_out)))
        return bad(GP_ERR_INVALID, "missing arrays or mismatched sizes");
    const int32_t n = usage->n_nodes, q = in->n_execs;
    if (n == 0) return bad(GP_ERR_INVALID, "empty node table");
    if (in->reserved_cpu_milli || in->reserved_mem_bytes || in->reserved_gpu)
        return bad(GP_ERR_INVALID, "reserved_* must be NULL (the overhead of the node table is the reserved amount)");
    const int32_t keep = scope ? scope->keep_topology_zone : -1;
    if (keep < -1) return bad(GP_ERR_INVALID, "scope->keep_topology_zone must be -1 or a zone id");
    if (keep >= 0) {
        if (!scope->topology_zone) return bad(GP_ERR_INVALID, "scope->topology_zone missing");
        for (int32_t i = 0; i < n; ++i)
            if (scope->topology_zone[i] < 0)
                return bad(GP_ERR_INVALID, "filterNodesToZone: a node has no topology.kubernetes.io/zone label (topology_zone == -1), "
                                           "unable to make scheduling decisions based on AZ");
    }
    if ((s = check_sort_ids(c, sort, who)) != GP_OK) return s;
    const bool mf = in->min_frag != 0;
    const bool has_host = mf && in->host_off;
    if ((s = check_requests(c, q, in->exe_cpu_milli, in->exe_mem_bytes, in->exe_gpu, who)) != GP_OK) return s;
    for (int32_t i = 0; i < q; ++i)
        if (in->group && in->group[i] != 0) return bad(GP_ERR_INVALID, "instance group out of range (one node table: group must be 0)");
    int64_t hosted = 0;
    if (has_host && (s = check_hosting(c, in, n, &hosted, who)) != GP_OK) return s;
    if (q == 0) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    // availability: one scatter of the reservations, one pass per node (usagebuf is scratch of the f2 stage only)
    long long *d_avail = nullptr, *d_sched = nullptr, *d_ff = nullptr;
    const long long* d_over[3] = {nullptr, nullptr, nullptr};
    int* d_err = nullptr;
    s = stage_availability(c, usage, st, &d_avail, &d_sched, &d_err, mf ? nullptr : &d_ff, d_over);
    if (s != GP_OK) return s;
    const size_t N = (size_t)n, Q = (size_t)q, H = (size_t)hosted, Z = (size_t)sort->n_zones;
    const bool zoned = sort->zone_id != nullptr && sort->n_zones > 1;
    Arena ar{c->reschedprep};
    const size_t o_tot = ar.take(8 * kZoneTotWords * Z), o_prio = ar.take(4 * Z), o_zone = ar.take(4 * N), o_nr = ar.take(4 * N), o_fu = ar.take(N),
                 o_fr = ar.take(N), o_lr = ar.take(4 * N), o_tz = ar.take(4 * N), o_rec = ar.take(sizeof(RpNode) * N), o_exe = ar.take(24 * Q),
                 o_hoff = ar.take(8 * (Q + 1)), o_hn = ar.take(4 * (H + 1)), o_out = ar.take(4 * Q), o_amb = ar.take(Q);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    if (zoned) GP_CUDA(c, ar.upload(o_zone, sort->zone_id, 4 * N, st));
    if (sort->name_rank) GP_CUDA(c, ar.upload(o_nr, sort->name_rank, 4 * N, st));
    if (sort->unschedulable) GP_CUDA(c, ar.upload(o_fu, sort->unschedulable, N, st));
    if (sort->ready) GP_CUDA(c, ar.upload(o_fr, sort->ready, N, st));
    if (sort->executor_label_rank) GP_CUDA(c, ar.upload(o_lr, sort->executor_label_rank, 4 * N, st));
    if (keep >= 0) GP_CUDA(c, ar.upload(o_tz, scope->topology_zone, 4 * N, st));
    GP_CUDA(c, ar.upload(o_exe, in->exe_cpu_milli, 8 * Q, st));
    GP_CUDA(c, ar.upload(o_exe + 8 * Q, in->exe_mem_bytes, 8 * Q, st));
    if (in->exe_gpu) GP_CUDA(c, ar.upload(o_exe + 16 * Q, in->exe_gpu, 8 * Q, st));
    else GP_CUDA(c, cudaMemsetAsync(b + o_exe + 16 * Q, 0, 8 * Q, st));
    if (has_host) {
        GP_CUDA(c, ar.upload(o_hoff, in->host_off, 8 * (Q + 1), st));
        if (H) GP_CUDA(c, ar.upload(o_hn, in->host_nodes, 4 * H, st));
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int32_t* tz = keep >= 0 ? (const int32_t*)(b + o_tz) : nullptr;
    if (zoned) {
        GP_CUDA(c, cudaMemsetAsync(b + o_tot, 0, 8 * kZoneTotWords * Z, st));
        gp_rp_zone_totals<<<nb, T, 0, st>>>(n, d_avail, d_avail + N, (const int32_t*)(b + o_zone), keep, tz, (unsigned long long*)(b + o_tot));
        gp_zone_priority<<<(sort->n_zones + T - 1) / T, T, 0, st>>>(sort->n_zones, (const unsigned long long*)(b + o_tot), (int32_t*)(b + o_prio));
    }
    RpNodeIn ni{};
    ni.avail = d_avail; ni.ff = d_ff;
    for (int d = 0; d < 3; ++d) ni.over[d] = d_over[d];
    ni.zone = zoned ? (const int32_t*)(b + o_zone) : nullptr;
    ni.prio = (const int32_t*)(b + o_prio);
    ni.name_rank = sort->name_rank ? (const int32_t*)(b + o_nr) : nullptr;
    ni.unschedulable = sort->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr;
    ni.ready = sort->ready ? (const uint8_t*)(b + o_fr) : nullptr;
    ni.label_rank = sort->executor_label_rank ? (const int32_t*)(b + o_lr) : nullptr;
    ni.tz = tz; ni.keep = keep; ni.n = n; ni.err = d_err;
    RpNode* rec = (RpNode*)(b + o_rec);
    gp_rp_nodes<<<nb, T, 0, st>>>(ni, rec);
    RpDecideIn di{};
    di.exe = (const int64_t*)(b + o_exe);
    di.host_off = has_host ? (const int64_t*)(b + o_hoff) : nullptr;
    di.host_nodes = (const int32_t*)(b + o_hn);
    di.n = n; di.q = q;
    // one CTA per executor; the grid is capped at 8 CTAs per SM's worth of executors and grid-strides over the rest.  The cap
    // only sizes the grid: registers bound residency (gp_rp_decide<true>: 78 x 256 threads -> 3 CTAs per SM; <false>: 48 -> 5),
    // so the CTAs beyond that wait for a free slot
    const int blocks = (int)std::min<int64_t>(q, (int64_t)c->sm_count * 8);
    int32_t* d_out = (int32_t*)(b + o_out);
    uint8_t* d_amb = ambiguous ? (uint8_t*)(b + o_amb) : nullptr;
    if (mf) gp_rp_decide<true><<<blocks, kRpThreads, 0, st>>>(rec, di, d_out, d_amb);
    else gp_rp_decide<false><<<blocks, kRpThreads, 0, st>>>(rec, di, d_out, d_amb);
    GP_CUDA(c, cudaGetLastError());
    GP_CUDA(c, cudaMemcpyAsync(node_out, d_out, 4 * Q, cudaMemcpyDeviceToHost, st));
    if (ambiguous) GP_CUDA(c, cudaMemcpyAsync(ambiguous, d_amb, Q, cudaMemcpyDeviceToHost, st));
    int err = 0;
    GP_CUDA(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return usage_refusal(c, err, who);                  // refused: node_out / ambiguous hold no decision
}

// the failover reconciler's findNodes loop for a batch of stale drivers (EXT/failover.go:43-82, 286-436); see
// gangpack_reconcile.cuh and DESIGN §2.3
gp_status gp_reconcile_find_nodes(gp_ctx* c, const gp_usage_input* usage, const gp_reconcile_nodes* nodes, const gp_apps* a,
                                  gp_reconcile_results* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_reconcile_find_nodes";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!nodes || !a || !out || nodes->n_groups < 1 || a->n_apps < 0 || (usage->n_nodes > 0 && (!nodes->node_group || !nodes->creation)) ||
        (a->n_apps > 0 && (!a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !out->placed)))
        return bad(GP_ERR_INVALID, "missing arrays or bad sizes (n_groups >= 1)");
    const int32_t n = usage->n_nodes, q = a->n_apps, G = nodes->n_groups;
    for (int32_t i = 0; i < n; ++i)
        if (nodes->node_group[i] < 0 || nodes->node_group[i] >= G) return bad(GP_ERR_INVALID, "node_group out of range");
    if ((s = check_requests(c, q, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu, who)) != GP_OK) return s;
    int64_t total = 0;
    for (int32_t i = 0; i < q; ++i) {
        const int32_t k = a->exe_count[i];
        if (k < 0) return bad(GP_ERR_INVALID, "negative exe_count");
        if (k > kMaxCount) return bad(GP_ERR_UNREPRESENTABLE, "exe_count > 2^24");
        if (a->group && (a->group[i] < 0 || a->group[i] >= G)) return bad(GP_ERR_INVALID, "instance group out of range");
        if (a->exec_out_off && a->exec_out_off[i] != total) return bad(GP_ERR_INVALID, "exec_out_off is not the prefix sum of exe_count");
        total += k;
    }
    if (a->exec_out_off && a->exec_out_off[q] != total) return bad(GP_ERR_INVALID, "exec_out_off is not the prefix sum of exe_count");
    if (total > 0 && (!out->executor_nodes || out->executor_nodes_cap < total))
        return bad(GP_ERR_CAPACITY, "executor_nodes_cap below the sum of exe_count");
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
    s = stage_availability(c, usage, st, &d_avail, &d_sched, &d_err);
    if (s != GP_OK) return s;
    const size_t N = (size_t)n, Q = (size_t)q, Gs = (size_t)G, E = (size_t)total;
    Arena ar{c->reconbuf};
    const size_t o_grp = ar.take(4 * N), o_cre = ar.take(8 * N), o_fu = ar.take(N), o_fr = ar.take(N), o_keys = ar.take(sizeof(ReconKey) * N),
                 o_sorted = ar.take(sizeof(ReconKey) * N), o_pos = ar.take(4 * N), o_order = ar.take(4 * N), o_ngrp = ar.take(4 * N),
                 o_noff = ar.take(4 * (Gs + 1)), o_aoff = ar.take(4 * (Gs + 1)), o_exe = ar.take(24 * Q), o_cnt = ar.take(4 * Q),
                 o_agrp = ar.take(4 * Q), o_off = ar.take(8 * Q), o_list = ar.take(4 * Q), o_lk = ar.take(sizeof(LabelKey) * Q),
                 o_lks = ar.take(sizeof(LabelKey) * Q), o_apos = ar.take(4 * Q), o_apps = ar.take(4 * Q), o_placed = ar.take(4 * Q),
                 o_exn = ar.take(4 * E), o_word = ar.take(16);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, ar.upload(o_grp, nodes->node_group, 4 * N, st));
    GP_CUDA(c, ar.upload(o_cre, nodes->creation, 8 * N, st));
    if (nodes->unschedulable) GP_CUDA(c, ar.upload(o_fu, nodes->unschedulable, N, st));
    if (nodes->ready) GP_CUDA(c, ar.upload(o_fr, nodes->ready, N, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_word, 0, 16, st));  // claim counter, error word
    if (!c->recon_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<ReconKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(ReconKey))));
        c->recon_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    ReconKey* keys = (ReconKey*)(b + o_keys);
    int32_t* pos = (int32_t*)(b + o_pos);
    int32_t* order = (int32_t*)(b + o_order);
    int32_t* ngrp = (int32_t*)(b + o_ngrp);
    gp_rc_node_keys<<<nb, T, 0, st>>>(n, G, (const int32_t*)(b + o_grp), (const long long*)(b + o_cre),
                                      nodes->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr, nodes->ready ? (const uint8_t*)(b + o_fr) : nullptr,
                                      keys, ngrp);
    gp_sort_tiles<ReconKey><<<(n + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(ReconKey), st>>>(n, nullptr, keys, (ReconKey*)(b + o_sorted));
    gp_rank_by_search<ReconKey><<<nb, T, 0, st>>>(n, nullptr, keys, (const ReconKey*)(b + o_sorted), pos);
    gp_scatter_order<<<nb, T, 0, st>>>(n, pos, order);
    int32_t* apps = (int32_t*)(b + o_apps);
    int32_t* agrp = (int32_t*)(b + o_agrp);
    int32_t* cnt = (int32_t*)(b + o_word + 8);
    if (q > 0) {
        // exe cpu, mem, gpu columns, counts, groups and offsets
        GP_CUDA(c, ar.upload(o_exe, a->exe_cpu_milli, 8 * Q, st));
        GP_CUDA(c, ar.upload(o_exe + 8 * Q, a->exe_mem_bytes, 8 * Q, st));
        if (a->exe_gpu) GP_CUDA(c, ar.upload(o_exe + 16 * Q, a->exe_gpu, 8 * Q, st));
        else GP_CUDA(c, cudaMemsetAsync(b + o_exe + 16 * Q, 0, 8 * Q, st));
        GP_CUDA(c, ar.upload(o_cnt, a->exe_count, 4 * Q, st));
        if (a->group) GP_CUDA(c, ar.upload(o_agrp, a->group, 4 * Q, st));
        else GP_CUDA(c, cudaMemsetAsync(agrp, 0, 4 * Q, st));
        if (a->exec_out_off) GP_CUDA(c, ar.upload(o_off, a->exec_out_off, 8 * Q, st));
        else {
            std::vector<int64_t>& off = c->host_off;
            off.resize(Q);
            int64_t run = 0;
            for (int32_t i = 0; i < q; ++i) { off[i] = run; run += a->exe_count[i]; }
            GP_CUDA(c, ar.upload(o_off, off.data(), 8 * Q, st));
        }
        // the stale drivers partitioned by group, call order kept inside each group
        const int qb = (q + T - 1) / T;
        gp_rc_app_list<<<qb, T, 0, st>>>(q, (int32_t*)(b + o_list), cnt);
        launch_label_resort(q, cnt, (const int32_t*)(b + o_list), agrp, (LabelKey*)(b + o_lk), (LabelKey*)(b + o_lks), (int32_t*)(b + o_apos),
                            apps, st);
    }
    gp_rc_offsets<<<(unsigned)((Gs + T) / T), T, 0, st>>>(G, n, order, ngrp, q, apps, agrp, (int32_t*)(b + o_noff), (int32_t*)(b + o_aoff));
    if (q > 0) {
        RcLoopIn li{};
        li.avail = d_avail; li.order = order; li.noff = (const int32_t*)(b + o_noff);
        li.apps = apps; li.aoff = (const int32_t*)(b + o_aoff);
        li.exe = (const long long*)(b + o_exe); li.count = (const int32_t*)(b + o_cnt); li.out_off = (const long long*)(b + o_off);
        li.placed = (int32_t*)(b + o_placed); li.exec_nodes = (int32_t*)(b + o_exn);
        li.claim = (unsigned int*)(b + o_word); li.err = (int*)(b + o_word + 4);
        li.n = n; li.q = q; li.n_groups = G;
        // one CTA per instance group; CTAs that find no group left return at once
        const int blocks = (int)std::min<int64_t>(G, (int64_t)c->sm_count * 8);
        gp_rc_loop<<<blocks, kRcThreads, 0, st>>>(li);
    }
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    if (q > 0) {
        GP_CUDA(c, cudaMemcpyAsync(out->placed, b + o_placed, 4 * Q, cudaMemcpyDeviceToHost, st));
        if (E) GP_CUDA(c, cudaMemcpyAsync(out->executor_nodes, b + o_exn, 4 * E, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(&herr, b + o_word + 4, 4, cudaMemcpyDeviceToHost, st));
    }
    int64_t* outs[3] = {out->avail_cpu_milli, out->avail_mem_bytes, out->avail_gpu};
    for (int d = 0; d < 3; ++d)
        if (outs[d]) GP_CUDA(c, cudaMemcpyAsync(outs[d], d_avail + N * (size_t)d, 8 * N, cudaMemcpyDeviceToHost, st));
    int uerr = 0;
    GP_CUDA(c, cudaMemcpyAsync(&uerr, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if ((s = usage_refusal(c, uerr, who)) != GP_OK) return s;
    if (herr & kRcErrDomain) return bad(GP_ERR_UNREPRESENTABLE, "an availability the loop charged lies outside the exact-int64 domain (|v| >= 2^61)");
    return GP_OK;
}

}  // extern "C"
