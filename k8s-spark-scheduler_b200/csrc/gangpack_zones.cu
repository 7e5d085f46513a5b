// gangpack_zones.cu -- the single-AZ and az-aware-tightly-pack packers (gp_pack_batch_zones, gp_pack_fifo_zones,
// gp_pack_fifo_az_aware, gp_pack_batch_az_aware) with gp_set_schedulable, the reservation table and usage deltas of the
// resident snapshot (gp_reserve_placements, gp_apply_usage_delta), and gp_packing_efficiency.
#include "gangpack_ctx.cuh"
#include "gangpack_zones.cuh"
#include "gangpack_zonefifo.cuh"
#include "gangpack_efficiency.cuh"

#include <algorithm>
#include <string>
#include <vector>

extern "C" {

// ---- single-AZ packers: pack every zone, choose by packing efficiency on the device (gangpack_zones.cuh) ----------
gp_status gp_set_schedulable(gp_ctx* c, const int64_t* cpu, const int64_t* mem, const int64_t* gpu) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_set_schedulable: gp_set_snapshot first");
    if (c->n_nodes > 0 && (!cpu || !mem)) return fail(c, GP_ERR_INVALID, "gp_set_schedulable: missing arrays");
    GP_CUDA(c, cudaSetDevice(c->device));
    const size_t N = (size_t)c->n_nodes;
    for (size_t i = 0; i < N; ++i) {
        const int64_t v[3] = {cpu[i], mem[i], gpu ? gpu[i] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_set_schedulable: |quantity| >= 2^61");
    }
    GP_CUDA(c, c->sched.reserve(24 * (N + 1)));
    char* b = c->sched.as<char>();
    if (N) {
        GP_CUDA(c, cudaMemcpyAsync(b, cpu, 8 * N, cudaMemcpyHostToDevice, c->stream));
        GP_CUDA(c, cudaMemcpyAsync(b + 8 * N, mem, 8 * N, cudaMemcpyHostToDevice, c->stream));
        if (gpu) GP_CUDA(c, cudaMemcpyAsync(b + 16 * N, gpu, 8 * N, cudaMemcpyHostToDevice, c->stream));
        else GP_CUDA(c, cudaMemsetAsync(b + 16 * N, 0, 8 * N, c->stream));
    }
    GP_CUDA(c, cudaStreamSynchronize(c->stream));
    c->have_sched = true;
    c->have_eff_sched = true;
    return GP_OK;
}

// ---- staging shared by the zone entry points ------------------------------------------------------------------------
// the arrays a non-empty batch of a zone entry point needs
static bool has_zone_arrays(const gp_apps* a, const gp_zone_results* out) {
    return a->drv_cpu_milli && a->drv_mem_bytes && a->exe_cpu_milli && a->exe_mem_bytes && a->exe_count && out->zone && out->driver_node;
}

// The six int64 quantity columns (6 x n_apps from o_in; absent gpu columns stay NULL = 0 in `six`), exe_count to o_cnt
// and the ExecutorNodes offsets `off` to o_off
static gp_status upload_app_columns(gp_ctx* c, const gp_apps* a, const int64_t* off, char* b, size_t o_in, size_t o_cnt, size_t o_off,
                                    cudaStream_t st, SixCols* six) {
    const size_t q = (size_t)a->n_apps;
    const int64_t* hc[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    *six = SixCols{};
    for (int k = 0; k < 6; ++k) {
        if (!hc[k]) continue;
        int64_t* d = reinterpret_cast<int64_t*>(b + o_in) + q * (size_t)k;
        GP_CUDA(c, cudaMemcpyAsync(d, hc[k], 8 * q, cudaMemcpyHostToDevice, st));
        six->p[k] = d;
    }
    GP_CUDA(c, cudaMemcpyAsync(b + o_cnt, a->exe_count, 4 * q, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_off, off, 8 * (q + 1), cudaMemcpyHostToDevice, st));
    return GP_OK;
}

// az-aware-tightly-pack: upload the undivided orders and build the fallback's gather view of them (gp_build_fallback_view).
// on_device: az's orders are device arrays (gp_prepare_cluster_zones' held orders) and are read in place.
static gp_status stage_fallback_view(gp_ctx* c, const gp_az_orders* az, bool on_device, cudaStream_t st, GatherSlots* fb) {
    const size_t ne = (size_t)az->n_exec, nd = (size_t)az->n_drv;
    Arena ar{c->fbview};
    const size_t o_eord = ar.take(on_device ? 0 : 4 * ne), o_dord = ar.take(on_device ? 0 : 4 * nd), o_npos = ar.take(4 * (size_t)c->n_nodes),
                 o_fbe = ar.take(4 * ne), o_fbd = ar.take(4 * nd), o_fbp = ar.take(4 * nd);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    const int32_t* eord = on_device ? az->exec_order : (const int32_t*)(b + o_eord);
    const int32_t* dord = on_device ? az->drv_order : (const int32_t*)(b + o_dord);
    if (!on_device && ne) GP_CUDA(c, cudaMemcpyAsync(b + o_eord, az->exec_order, 4 * ne, cudaMemcpyHostToDevice, st));
    if (!on_device && nd) GP_CUDA(c, cudaMemcpyAsync(b + o_dord, az->drv_order, 4 * nd, cudaMemcpyHostToDevice, st));
    gp_build_fallback_view<<<1, 1024, 0, st>>>(c->n_nodes, (int32_t)ne, (int32_t)nd, eord, dord,
                                               c->node_slot.as<int32_t>(), (int32_t*)(b + o_npos), (int32_t*)(b + o_fbe), (int32_t*)(b + o_fbd),
                                               (int32_t*)(b + o_fbp));
    c->last.kernel_launches += 1;
    *fb = GatherSlots{(const int32_t*)(b + o_fbe), (const int32_t*)(b + o_fbd), (const int32_t*)(b + o_fbp), (int32_t)ne, (int32_t)nd};
    return GP_OK;
}

// zone / driver / ExecutorNodes (T entries) / averages to the host, one synchronise, then the kernels' validation errors
static gp_status finish_zone_results(gp_ctx* c, gp_zone_results* out, const int32_t* zone, const int32_t* drv, const int32_t* exe,
                                     const double* avg, size_t q, size_t T, cudaStream_t st) {
    GP_CUDA(c, cudaMemcpyAsync(out->zone, zone, 4 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(out->driver_node, drv, 4 * q, cudaMemcpyDeviceToHost, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(out->executor_nodes, exe, 4 * T, cudaMemcpyDeviceToHost, st));
    if (out->avg_efficiency) GP_CUDA(c, cudaMemcpyAsync(out->avg_efficiency, avg, 32 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return host_error(c);
}

// Independent zone packs of a batch, shared by gp_pack_batch_zones (the zones are every instance group, no fallback) and
// gp_pack_batch_az_aware (zones 0..Z-1 with tightly-pack, plus the undivided orders `az` of the fallback, already
// validated; az_dev: they are device arrays).  Argument checks common to both are here.
static gp_status batch_zones_run(gp_ctx* c, const gp_apps* a, gp_algo algo, int32_t Z, const gp_az_orders* az, bool az_dev,
                                 gp_zone_results* out, const char* who) {
    const std::string w(who);
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, w + ": missing app/result arrays");
    if ((int64_t)Q * Z > 0x7fffffffLL) return fail(c, GP_ERR_INVALID, w + ": n_apps x zones too large");
    const int64_t* off = a->exec_out_off;
    if (!off) {
        c->host_off.resize((size_t)Q + 1);
        int64_t acc = 0;
        for (int32_t i = 0; i < Q; ++i) { c->host_off[(size_t)i] = acc; acc += a->exe_count[i] > 0 ? a->exe_count[i] : 0; }
        c->host_off[(size_t)Q] = acc;
        off = c->host_off.data();
    }
    const int64_t total = off[Q];
    if (total < 0 || total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, w + ": executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, w + ": executor_nodes is NULL");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, R = q * (size_t)Z, T = (size_t)total;
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_rows = ar.take(48 * R), o_rcnt = ar.take(4 * R),
                 o_rgrp = ar.take(4 * R), o_roff = ar.take(8 * (R + 1)), o_rdrv = ar.take(4 * R), o_rexe = ar.take(4 * ((size_t)Z * T + 1)),
                 o_zone = ar.take(4 * q), o_drv = ar.take(4 * q), o_exe = ar.take(4 * (T + 1)), o_avg = ar.take(32 * q);
    // az-aware: the fallback's PrepApp records and list
    const size_t QF = az ? q : 0;
    const size_t o_prep = ar.take(sizeof(PrepApp) * QF), o_list = ar.take(4 * QF);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    SixCols six;
    gp_status s = upload_app_columns(c, a, off, b, o_in, o_cnt, o_off, st, &six);
    if (s != GP_OK) return s;
    const int TH = 256;
    // the efficiencies read the availability in node-table order: refresh that copy from the slots (a FIFO batch may
    // have charged them since gp_set_snapshot)
    if (c->n_slots > 0)
        gp_scatter_slots<<<(c->n_slots + TH - 1) / TH, TH, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(), c->slot_node.as<int32_t>(),
                                                                   c->node_cpu.as<int64_t>(), c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
    gp_zone_expand<<<(unsigned)((R + 1 + TH - 1) / TH), TH, 0, st>>>(Q, Z, six, (const int32_t*)(b + o_cnt), (const int64_t*)(b + o_off),
                                                                      (int64_t*)(b + o_rows), (int32_t*)(b + o_rcnt), (int32_t*)(b + o_rgrp), (int64_t*)(b + o_roff));
    int2* scratch = nullptr;
    s = pack_begin(c, (int32_t)R, algo, GP_MODE_INDEPENDENT, (int64_t)Z * total, false, &scratch, st);
    if (s != GP_OK) return s;
    DevApps dv{};
    for (int k = 0; k < 6; ++k) dv.cols.q[k] = b + o_rows + 8 * R * (size_t)k;
    dv.cols.count = (const int32_t*)(b + o_rcnt); dv.cols.group = (const int32_t*)(b + o_rgrp); dv.cols.off = (const int64_t*)(b + o_roff);
    dv.cols.bits = 64; dv.cols.mem_shift = 0; dv.skip = nullptr; dv.n = (int32_t)R;
    DevResults dr{(int32_t*)(b + o_rdrv), b + o_rexe, (int64_t)Z * total, 32};
    s = pack_device_range(c, dv, 0, (int32_t)R, 0, algo, GP_MODE_INDEPENDENT, dr, scratch, st, 0);
    if (s != GP_OK) return s;
    c->ev_chunks = 1;
    ZoneChooseIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.avail[0] = c->node_cpu.as<long long>(); zi.avail[1] = c->node_mem.as<long long>(); zi.avail[2] = c->node_gpu.as<long long>();
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    for (int k = 0; k < 3; ++k) { zi.drv[k] = six.p[k]; zi.exe[k] = six.p[3 + k]; }
    zi.count = (const int32_t*)(b + o_cnt); zi.out_off = (const int64_t*)(b + o_off);
    zi.row_driver = (const int32_t*)(b + o_rdrv); zi.row_exec = (const int32_t*)(b + o_rexe);
    zi.n_apps = Q; zi.n_zones = Z; zi.executors_reserved = algo == GP_TIGHTLY_PACK ? 1 : 0;
    gp_zone_choose<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(zi, (int32_t*)(b + o_zone), (int32_t*)(b + o_drv), (int32_t*)(b + o_exe),
                                                                       out->avg_efficiency ? (double*)(b + o_avg) : nullptr);
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    if (az) {
        // the applications no zone won: SparkBinPack(tightlyPackExecutors) over the undivided orders, still on the device
        // (az_aware_pack_tightly.go:33-37).  The list length and the fallback's claim counter are zeroed by pack_begin;
        // stats [2..3] restart so that scan_path_apps / _nodes count the fallback alone.
        DevStatus* ds = c->status();
        unsigned long long* d_stats = ds->head.stats;
        GP_CUDA(c, cudaMemsetAsync(d_stats + 2, 0, 16, st));
        int32_t* listed = (int32_t*)(b + o_list);
        gp_az_fallback_list<<<(unsigned)((q + TH - 1) / TH), TH, 0, st>>>(Q, (const int32_t*)(b + o_zone), listed, &ds->az_listed);
        AppColumns cols{};
        for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
        cols.count = (const int32_t*)(b + o_cnt); cols.group = nullptr; cols.off = (const int64_t*)(b + o_off); cols.bits = 64; cols.mem_shift = 0;
        PrepApp* prep = (PrepApp*)(b + o_prep);
        gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
            Q, cols, nullptr, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, prep, &ds->head.err, &c->host_status()->err_word);
        GatherSlots fb;
        s = stage_fallback_view(c, az, az_dev, st, &fb);
        if (s != GP_OK) return s;
        int& per_sm = c->az_fallback_ctas_per_sm;
        if (per_sm == 0) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_pack_az_fallback, kAzFallbackThreads, 0);
            if (per_sm < 1) per_sm = 1;
        }
        int64_t blocks = ((int64_t)Q * 32 + kAzFallbackThreads - 1) / kAzFallbackThreads;   // the list holds at most Q
        if (blocks > (int64_t)c->sm_count * per_sm) blocks = (int64_t)c->sm_count * per_sm;
        gp_pack_az_fallback<<<(unsigned)blocks, kAzFallbackThreads, 0, st>>>(make_snapshot(c), prep, listed, &ds->az_listed, fb, (int32_t*)(b + o_drv),
                                                                            (int32_t*)(b + o_exe), d_stats, &ds->az_claim);
        GP_CUDA(c, cudaGetLastError());
        c->last.kernel_launches += 3;
    }
    return finish_zone_results(c, out, (const int32_t*)(b + o_zone), (const int32_t*)(b + o_drv), (const int32_t*)(b + o_exe),
                               (const double*)(b + o_avg), q, T, st);
}

gp_status gp_pack_batch_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_batch_zones: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: the single-AZ packers are tightly-pack and minimal-fragmentation (single_az_pack_tightly.go, single_az_minimal_fragmentation.go)");
    return batch_zones_run(c, a, algo, c->n_groups, nullptr, false, out, "gp_pack_batch_zones");
}

// ---- reservation table + device-resident snapshot upkeep (gangpack_zones.cuh) -------------------------------------------
static gp_status refresh_views(gp_ctx* c, cudaStream_t st) {
    const int T = 256;
    if (c->n_slots <= 0) return GP_OK;
    SnapMeta* meta = c->snap_flags.as<SnapMeta>();
    gp_refresh_meta<<<(c->n_slots + T - 1) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->slot_node.as<int32_t>(),
                                                           &meta->flags, meta->max_avail);
    gp_fill_pair32<<<(c->n_slots + T) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), meta, c->pair32.as<uint2>());
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// The undivided orders of az-aware-tightly-pack against the snapshot gp_set_snapshot laid out, in O(N): every entry a node
// of the snapshot in that role, once; every zone group's order = the undivided order restricted to that group's nodes
// (the fallback and the zone packs must see the same priorities).  o->n_zones is already within 0..n_groups.
static gp_status check_az_orders(gp_ctx* c, const gp_az_orders* o, const char* who) {
    const std::string w(who);
    if (!c->host_layout)
        return fail(c, GP_ERR_INVALID, w + ": the snapshot must be laid out by gp_set_snapshot (after gp_set_snapshot_device / "
                                           "gp_prepare_cluster there is no host copy of the layout to check the undivided orders against)");
    if (o->n_exec != c->n_exec || o->n_drv != c->n_drv)
        return fail(c, GP_ERR_INVALID, w + ": order lengths must equal the snapshot's exec_off[n_groups] / drv_off[n_groups]");
    if ((o->n_exec > 0 && !o->exec_order) || (o->n_drv > 0 && !o->drv_order))
        return fail(c, GP_ERR_INVALID, w + ": order arrays missing");
    const int32_t Z = o->n_zones;
    const uint32_t N = (uint32_t)c->n_nodes;
    const int32_t* owner = c->v_owner.data();
    const int32_t* pos = c->v_pos.data();
    for (int role = 0; role < 2; ++role) {
        const int32_t n = role == 0 ? o->n_exec : o->n_drv;
        const int32_t* ord = role == 0 ? o->exec_order : o->drv_order;
        const char* name = role == 0 ? "exec_order" : "drv_order";
        std::vector<uint8_t>& seen = role == 0 ? c->v_seen_e : c->v_seen_d;
        seen.assign((size_t)N, 0);
        std::vector<int32_t>& next = c->v_zone_next;     // next expected position in each zone group's order
        next.assign((size_t)Z, 0);
        for (int32_t i = 0; i < n; ++i) {
            const uint32_t v = (uint32_t)ord[i];
            if (v >= N) return fail(c, GP_ERR_INVALID, w + ": " + name + " entry out of range");
            if (seen[v]) return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node twice");
            seen[v] = 1;
            const int32_t ow = owner[v];
            if (ow < 0 || !(ow & (1 << role)))
                return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node the snapshot does not list as " +
                                                   (role == 0 ? "an executor" : "a driver") + " candidate");
            const int32_t g = ow >> 2;
            if (g < Z && pos[(size_t)role * N + v] != next[(size_t)g]++)
                return fail(c, GP_ERR_INVALID, w + ": zone group " + std::to_string(g) + "'s " +
                                                   (role == 0 ? "executor" : "driver") + " order is not " + name + " restricted to its nodes");
        }
    }
    return GP_OK;
}

// The az-aware entries' NULL arguments.  orders == NULL stands for the undivided orders and n_zones gp_prepare_cluster_zones
// (GP_LAYOUT_AZ_AWARE) left on the device -- *o then points at them; after any other snapshot it is refused.
static gp_status held_az_orders(gp_ctx* c, const gp_apps* a, const gp_zone_results* out, const gp_az_orders** o, const char* who) {
    const std::string w(who);
    if (!*o && c->zone_kind == GP_LAYOUT_SINGLE_AZ)
        return fail(c, GP_ERR_INVALID, w + ": orders == NULL needs a gp_prepare_cluster_zones(GP_LAYOUT_AZ_AWARE) snapshot; this one is "
                                           "GP_LAYOUT_SINGLE_AZ (no trailing group, no undivided orders)");
    if (!a || !out || (!*o && c->zone_kind != GP_LAYOUT_AZ_AWARE) || a->n_apps < 0) return fail(c, GP_ERR_INVALID, w + ": NULL apps/orders/results");
    if (!*o) *o = &c->zone_orders;
    return GP_OK;
}

// The FIFO loop over zones in one launch (gangpack_zonefifo.cuh), shared by gp_pack_fifo_zones (kind = 0 tightly-pack,
// 2 minimal-fragmentation; the zones are every instance group) and gp_pack_fifo_az_aware (kind = kZoneAzAware; zones
// 0..Z-1, plus the undivided orders `az` of the fallback, already validated; az_dev: they are device arrays).  Argument
// checks common to both are here.
static gp_status fifo_zones_run(gp_ctx* c, const gp_apps* a, int kind, gp_mode mode, int32_t Z, const gp_az_orders* az, bool az_dev,
                                gp_zone_results* out, const char* who) {
    const std::string w(who);
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, w + ": missing app/result arrays");
    std::vector<int64_t>& hoff = c->host_off;
    hoff.resize((size_t)Q + 1);
    int64_t acc = 0, pitch = 1;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        hoff[(size_t)i] = acc; acc += k;
        if (k > pitch) pitch = k;
    }
    hoff[(size_t)Q] = acc;
    if (a->exec_out_off)
        for (int32_t i = 0; i <= Q; ++i)
            if (a->exec_out_off[i] != hoff[(size_t)i]) return fail(c, GP_ERR_INVALID, w + ": exec_out_off must be the prefix sum of exe_count (or NULL)");
    const int64_t total = acc;
    if (total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, w + ": executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, w + ": executor_nodes is NULL");
    pitch = (pitch + 3) & ~(int64_t)3;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const bool azk = kind == kZoneAzAware;
    const size_t q = (size_t)Q, T = (size_t)total, RP = (size_t)(Z + (azk ? 1 : 0)) * (size_t)pitch;   // az-aware: row Z = fallback
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_skip = ar.take(q), o_rexe = ar.take(4 * RP),
                 o_rlist = ar.take(kind == GP_MINIMAL_FRAGMENTATION ? 8 * RP : 0), o_zone = ar.take(4 * q), o_drv = ar.take(4 * q),
                 o_exe = ar.take(4 * (T + 1)), o_avg = ar.take(32 * q);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    int2* unused = nullptr;
    gp_status s = pack_begin(c, Q, GP_TIGHTLY_PACK, mode, total, false, &unused, st);
    if (s != GP_OK) return s;
    SixCols six;
    s = upload_app_columns(c, a, hoff.data(), b, o_in, o_cnt, o_off, st, &six);
    if (s != GP_OK) return s;
    if (a->skip_if_no_fit) GP_CUDA(c, cudaMemcpyAsync(b + o_skip, a->skip_if_no_fit, q, cudaMemcpyHostToDevice, st));
    AppColumns cols{};
    for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
    cols.count = (const int32_t*)(b + o_cnt); cols.group = nullptr; cols.off = (const int64_t*)(b + o_off); cols.bits = 64; cols.mem_shift = 0;
    DevStatus* ds = c->status();
    unsigned long long* d_stats = ds->head.stats;
    PrepApp* prep = c->prep.as<PrepApp>();
    gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
        Q, cols, a->skip_if_no_fit ? (const uint8_t*)(b + o_skip) : nullptr, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, prep,
        &ds->head.err, &c->host_status()->err_word);
    Snapshot snap = make_snapshot(c);
    ZoneFifoIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    zi.node_slot = c->node_slot.as<int32_t>();
    zi.row_exec = (int32_t*)(b + o_rexe);
    zi.row_list = kind == GP_MINIMAL_FRAGMENTATION ? (int2*)(b + o_rlist) : nullptr;
    zi.row_pitch = pitch; zi.n_apps = Q; zi.n_zones = Z;
    double* avg = out->avg_efficiency ? (double*)(b + o_avg) : nullptr;
    int32_t* zo = (int32_t*)(b + o_zone); int32_t* dq = (int32_t*)(b + o_drv); int32_t* eo = (int32_t*)(b + o_exe);
    GatherSlots fb{};
    if (azk) {
        s = stage_fallback_view(c, az, az_dev, st, &fb);
        if (s != GP_OK) return s;
    }
    if (kind == GP_TIGHTLY_PACK) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<0, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<0, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else if (kind == GP_MINIMAL_FRAGMENTATION) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<2, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<2, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<kZoneAzAware, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
        else gp_pack_fifo_zones_cta<kZoneAzAware, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
    }
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    s = refresh_views(c, st);                          // the compact view follows the charged slots
    if (s != GP_OK) return s;
    return finish_zone_results(c, out, zo, dq, eo, avg, q, T, st);
}

// the FIFO loop with a single-AZ packer in one launch
gp_status gp_pack_fifo_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_mode mode, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_fifo_zones: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: the single-AZ packers are tightly-pack and minimal-fragmentation");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones)");
    const int32_t Z = c->n_groups;
    if (Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: more than 64 zones");
    return fifo_zones_run(c, a, (int)algo, mode, Z, nullptr, false, out, "gp_pack_fifo_zones");
}

// the FIFO loop with az-aware-tightly-pack in one launch: the zone packs plus the undivided fallback on the device
gp_status gp_pack_fifo_az_aware(gp_ctx* c, const gp_apps* a, gp_mode mode, const gp_az_orders* o, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_fifo_az_aware: gp_set_snapshot first");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones, "
                                       "then gp_pack_batch over the undivided orders)");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    gp_status s = held_az_orders(c, a, out, &o, "gp_pack_fifo_az_aware");
    if (s != GP_OK) return s;
    const bool held = o == &c->zone_orders;
    const int32_t Z = o->n_zones;
    if (Z < 0 || Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones must be 0..64");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones exceeds the snapshot's instance groups");
    if (!held) s = check_az_orders(c, o, "gp_pack_fifo_az_aware");
    if (s != GP_OK) return s;
    return fifo_zones_run(c, a, kZoneAzAware, mode, Z, o, held, out, "gp_pack_fifo_az_aware");
}

// az-aware-tightly-pack for a batch of independent decisions: the zone packs, the zone choice and the undivided fallback
// on the device, one stream synchronise
gp_status gp_pack_batch_az_aware(gp_ctx* c, const gp_apps* a, const gp_az_orders* o, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_batch_az_aware: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    gp_status s = held_az_orders(c, a, out, &o, "gp_pack_batch_az_aware");
    if (s != GP_OK) return s;
    const bool held = o == &c->zone_orders;
    const int32_t Z = o->n_zones;
    if (Z < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones is negative");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones exceeds the snapshot's instance groups");
    if (!held) s = check_az_orders(c, o, "gp_pack_batch_az_aware");
    if (s != GP_OK) return s;
    return batch_zones_run(c, a, GP_TIGHTLY_PACK, Z, o, held, out, "gp_pack_batch_az_aware");
}

gp_status gp_reserve_placements(gp_ctx* c, const gp_apps* a, const gp_results* placed, int32_t subtract, gp_reservation_table* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_reserve_placements: gp_set_snapshot first");
    if (!a || !placed || a->n_apps < 0 || (!out && !subtract)) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: NULL arguments");
    const int32_t Q = a->n_apps;
    if (out) out->n_rows = 0;
    if (Q == 0) return GP_OK;
    if (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !placed->driver_node)
        return fail(c, GP_ERR_INVALID, "gp_reserve_placements: missing app/result arrays");
    // host pass: offsets, rows per placed application, index validation
    std::vector<int64_t>& off = c->host_off;
    off.resize(2 * ((size_t)Q + 1));
    int64_t* roff = off.data() + Q + 1;
    int64_t acc = 0, rows = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        off[(size_t)i] = a->exec_out_off ? a->exec_out_off[i] : acc;
        acc += k;
        roff[i] = rows;
        const int32_t d = placed->driver_node[i];
        if (d >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: driver_node out of range");
        if (d >= 0) {
            if (k > 0 && !placed->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: executor_nodes is NULL");
            if (off[(size_t)i] < 0 || off[(size_t)i] + k > placed->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, "gp_reserve_placements: offsets exceed executor_nodes_cap");
            for (int64_t t = 0; t < k; ++t) {
                const int32_t n = placed->executor_nodes[off[(size_t)i] + t];
                if (n < 0 || n >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: executor node out of range");
            }
            rows += 1 + k;
        }
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    roff[Q] = rows;
    const int64_t total = placed->executor_nodes_cap < off[(size_t)Q] ? placed->executor_nodes_cap : off[(size_t)Q];
    if (out && rows > out->rows_cap) return fail(c, GP_ERR_CAPACITY, "gp_reserve_placements: rows_cap too small");
    if (out && rows > 0 && (!out->app || !out->slot || !out->node || !out->cpu_milli || !out->mem_bytes))
        return fail(c, GP_ERR_INVALID, "gp_reserve_placements: missing table arrays");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)(total > 0 ? total : 0), R = (size_t)rows;
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_roff = ar.take(8 * (q + 1)), o_drv = ar.take(4 * q),
                 o_exe = ar.take(4 * (T + 1)), o_ra = ar.take(4 * (R + 1)), o_rs = ar.take(4 * (R + 1)), o_rn = ar.take(4 * (R + 1)),
                 o_rc = ar.take(8 * (R + 1)), o_rm = ar.take(8 * (R + 1)), o_rg = ar.take(8 * (R + 1));
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    ReserveIn ri{};
    gp_status s = upload_app_columns(c, a, off.data(), b, o_in, o_cnt, o_off, st, &ri.cols);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(b + o_roff, roff, 8 * (q + 1), cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_drv, placed->driver_node, 4 * q, cudaMemcpyHostToDevice, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(b + o_exe, placed->executor_nodes, 4 * T, cudaMemcpyHostToDevice, st));
    ri.count = (const int32_t*)(b + o_cnt); ri.off = (const int64_t*)(b + o_off); ri.row_off = (const int64_t*)(b + o_roff);
    ri.driver = (const int32_t*)(b + o_drv); ri.exec = (const int32_t*)(b + o_exe); ri.n_apps = Q; ri.subtract = subtract ? 1 : 0;
    ReserveOut ro{(int32_t*)(b + o_ra), (int32_t*)(b + o_rs), (int32_t*)(b + o_rn), (long long*)(b + o_rc), (long long*)(b + o_rm), (long long*)(b + o_rg)};
    const int TH = 256;
    gp_reserve_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, ro, c->node_slot.as<int32_t>(), c->pair.as<longlong2>(), c->sgpu.as<long long>(),
                                                                        c->node_cpu.as<long long>(), c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    if (subtract) { s = refresh_views(c, st); if (s != GP_OK) return s; }
    if (out && R) {
        GP_CUDA(c, cudaMemcpyAsync(out->app, ro.app, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->slot, ro.slot, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->node, ro.node, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->cpu_milli, ro.cpu, 8 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->mem_bytes, ro.mem, 8 * R, cudaMemcpyDeviceToHost, st));
        if (out->gpu) GP_CUDA(c, cudaMemcpyAsync(out->gpu, ro.gpu, 8 * R, cudaMemcpyDeviceToHost, st));
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (out) out->n_rows = rows;
    return GP_OK;
}

gp_status gp_apply_usage_delta(gp_ctx* c, int64_t n_rows, const int32_t* node, const int64_t* cpu, const int64_t* mem, const int64_t* gpu, int32_t sign) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_apply_usage_delta: gp_set_snapshot first");
    if (n_rows < 0 || (sign != 1 && sign != -1) || (n_rows > 0 && (!node || !cpu || !mem))) return fail(c, GP_ERR_INVALID, "gp_apply_usage_delta: bad arguments");
    if (n_rows == 0) return GP_OK;
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t v[3] = {cpu[r], mem[r], gpu ? gpu[r] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_apply_usage_delta: |quantity| >= 2^61");
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t R = (size_t)n_rows;
    Arena ar{c->zonebuf};
    const size_t o_c = ar.take(8 * R), o_m = ar.take(8 * R), o_g = ar.take(8 * R), o_n = ar.take(4 * R);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, cudaMemcpyAsync(b + o_c, cpu, 8 * R, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_m, mem, 8 * R, cudaMemcpyHostToDevice, st));
    if (gpu) GP_CUDA(c, cudaMemcpyAsync(b + o_g, gpu, 8 * R, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_n, node, 4 * R, cudaMemcpyHostToDevice, st));
    const int TH = 256;
    gp_usage_delta<<<(unsigned)((R + TH - 1) / TH), TH, 0, st>>>(n_rows, (const int32_t*)(b + o_n), (const long long*)(b + o_c), (const long long*)(b + o_m),
                                                                  gpu ? (const long long*)(b + o_g) : nullptr, sign, c->n_nodes, c->node_slot.as<int32_t>(),
                                                                  c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_cpu.as<long long>(),
                                                                  c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    gp_status s = refresh_views(c, st);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

// ---- computeAvgPackingEfficiencyForResult over the whole node table, exactly summed (gangpack_efficiency.cuh) ----------
gp_status gp_packing_efficiency(gp_ctx* c, const gp_apps* a, gp_algo algo, const gp_results* placed, gp_mode charged, double* avg_out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_packing_efficiency: no snapshot (gp_set_snapshot, gp_prepare_cluster or gp_prepare_cluster_zones first)");
    if (!c->have_eff_sched)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: no SchedulableResources (gp_set_schedulable, gp_prepare_cluster or gp_prepare_cluster_zones first)");
    if (!a || !placed || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: NULL apps/placed");
    if (algo != GP_TIGHTLY_PACK && algo != GP_DISTRIBUTE_EVENLY && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: unknown algo");
    if (charged != GP_MODE_INDEPENDENT && charged != GP_MODE_FIFO_REFERENCE && charged != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: unknown charged mode");
    if (charged != GP_MODE_INDEPENDENT && a->n_apps != 1)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: a FIFO charged mode adds back ONE application's usage: n_apps must be 1");
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!avg_out || !a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !placed->driver_node)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: missing app/result arrays");
    // host pass over the placed rows: offsets, request domain, node indices (a caller-supplied placement need not be feasible)
    std::vector<int64_t>& off = c->host_off;
    off.resize((size_t)Q + 1);
    const int64_t* qc[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    int64_t acc = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        off[(size_t)i] = a->exec_out_off ? a->exec_out_off[i] : acc;
        acc += k;
        const int32_t d = placed->driver_node[i];
        if (d >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: driver_node out of range");
        if (d < 0) continue;
        for (const int64_t* col : qc) {
            if (!col) continue;
            if (col[i] < 0) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: negative request");
            if (col[i] >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: request >= 2^61");
        }
        if (k > 0 && !placed->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: executor_nodes is NULL");
        if (off[(size_t)i] < 0 || off[(size_t)i] + k > placed->executor_nodes_cap)
            return fail(c, GP_ERR_CAPACITY, "gp_packing_efficiency: offsets exceed executor_nodes_cap");
        for (int64_t t = 0; t < k; ++t) {
            const int32_t n = placed->executor_nodes[off[(size_t)i] + t];
            if (n < 0 || n >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: executor node out of range");
        }
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    const int64_t total = placed->executor_nodes_cap < off[(size_t)Q] ? placed->executor_nodes_cap : off[(size_t)Q];
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)(total > 0 ? total : 0), N = (size_t)c->n_nodes;
    const int TH = kEffThreads;
    const int n_part = (int)std::max<size_t>(1, std::min<size_t>((N + TH - 1) / TH, (size_t)c->sm_count * 4));
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_drv = ar.take(4 * q), o_exe = ar.take(4 * (T + 1)),
                 o_part = ar.take(sizeof(EffAcc) * (size_t)n_part), o_base = ar.take(sizeof(EffAcc)), o_avg = ar.take(32 * q), o_err = ar.take(4);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    EffRowsIn ri{};
    gp_status s = upload_app_columns(c, a, off.data(), b, o_in, o_cnt, o_off, st, &ri.cols);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(b + o_drv, placed->driver_node, 4 * q, cudaMemcpyHostToDevice, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(b + o_exe, placed->executor_nodes, 4 * T, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_err, 0, 4, st));
    int* d_err = (int*)(b + o_err);
    EffBaseIn bi{};
    bi.av = SnapshotAvail{c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_slot.as<int32_t>(), c->node_cpu.as<long long>(),
                      c->node_mem.as<long long>(), c->node_gpu.as<long long>()};
    bi.sched[0] = c->sched.as<long long>(); bi.sched[1] = c->sched.as<long long>() + N; bi.sched[2] = c->sched.as<long long>() + 2 * N;
    bi.n_nodes = c->n_nodes;
    EffAcc* base = (EffAcc*)(b + o_base);
    gp_eff_base<<<n_part, TH, 0, st>>>(bi, (EffAcc*)(b + o_part), d_err);
    gp_eff_finish<<<1, TH, 0, st>>>((const EffAcc*)(b + o_part), n_part, base);
    ri.av = bi.av;
    for (int k = 0; k < 3; ++k) ri.sched[k] = bi.sched[k];
    ri.count = (const int32_t*)(b + o_cnt); ri.off = (const int64_t*)(b + o_off);
    ri.driver = (const int32_t*)(b + o_drv); ri.exec = (const int32_t*)(b + o_exe); ri.base = base;
    ri.n_apps = Q; ri.n_nodes = c->n_nodes;
    ri.executors_reserved = algo == GP_MINIMAL_FRAGMENTATION ? 0 : 1;
    ri.charged = (int32_t)charged;
    gp_eff_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, (double*)(b + o_avg), d_err);
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    GP_CUDA(c, cudaMemcpyAsync(avg_out, b + o_avg, 32 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (herr & kEffErrQuantity)
        return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: a per-node reserved amount is >= 2^61");
    if (herr & kEffErrRange)
        return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: an efficiency term outside the exact accumulator's range");
    return GP_OK;
}
}  // extern "C"
