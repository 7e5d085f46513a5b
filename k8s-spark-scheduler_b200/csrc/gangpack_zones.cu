// gangpack_zones.cu -- the single-AZ and az-aware-tightly-pack packers (gp_pack_batch_zones, gp_pack_fifo_zones,
// gp_pack_fifo_az_aware, gp_pack_batch_az_aware, gp_pack_fifo_zones_groups) with gp_set_schedulable, the reservation table and usage deltas of the
// resident snapshot (gp_reserve_placements, gp_apply_usage_delta), and gp_packing_efficiency[_groups].
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
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), "gp_set_schedulable"));
    if (c->n_nodes > 0 && (!cpu || !mem)) return fail(c, GP_ERR_INVALID, "gp_set_schedulable: missing arrays");
    GP_CUDA(c, cudaSetDevice(c->device));
    const size_t N = (size_t)c->n_nodes;
    for (size_t i = 0; i < N; ++i) {
        const int64_t v[3] = {cpu[i], mem[i], gpu ? gpu[i] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_set_schedulable: |quantity| >= 2^61");
    }
    Arena ar{c->sched, c->stream};
    const auto sched = ar.take<long long>(3 * (N + 1));
    ar.reserve();
    ar.put(sched.part(0, N), cpu);
    ar.put(sched.part(N, N), mem);
    ar.put_or_zero(sched.part(2 * N, N), gpu);
    GP_TRY(ar.sync(c));
    c->held.schedulable_set();
    return GP_OK;
}

// ---- staging shared by the zone entry points ------------------------------------------------------------------------
// the arrays a non-empty batch of a zone entry point needs
static bool has_zone_arrays(const gp_apps* a, const gp_zone_results* out) {
    return a->drv_cpu_milli && a->drv_mem_bytes && a->exe_cpu_milli && a->exe_mem_bytes && a->exe_count && out->zone && out->driver_node;
}

// Uploads the six int64 quantity columns (6 x n_apps of `in`; absent gpu columns stay NULL = 0 in the result), exe_count
// and the ExecutorNodes offsets `off`
static SixCols upload_app_columns(Arena& ar, const gp_apps* a, const int64_t* off, Piece<int64_t> in, Piece<int32_t> cnt,
                                  Piece<int64_t> d_off) {
    const size_t q = (size_t)a->n_apps;
    const int64_t* hc[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    SixCols six{};
    for (int k = 0; k < 6; ++k) six.p[k] = ar.put(in.part(q * k, q), hc[k]);
    ar.put(cnt, a->exe_count);
    ar.put(d_off, off);
    return six;
}

// One instance group over the whole snapshot (gp_pack_fifo_zones, gp_pack_*_az_aware) in the layout of
// gp_pack_fifo_zones_groups; o: the az-aware orders, NULL for the single-AZ packers
struct OneInstanceGroup {
    int32_t group_off[2], n_zones, exec_off[2], drv_off[2];
    gp_instance_groups ig;
    OneInstanceGroup(int32_t n_groups, const gp_az_orders* o)
        : group_off{0, n_groups}, n_zones(o ? o->n_zones : 0), exec_off{0, o ? o->n_exec : 0}, drv_off{0, o ? o->n_drv : 0},
          ig{1, group_off, o ? &n_zones : nullptr, o ? exec_off : nullptr, o ? o->exec_order : nullptr, o ? drv_off : nullptr,
             o ? o->drv_order : nullptr} {}
    OneInstanceGroup(const OneInstanceGroup&) = delete;
    OneInstanceGroup& operator=(const OneInstanceGroup&) = delete;
};

// az-aware-tightly-pack: upload the undivided orders of the instance groups `ig` and build the fallback's gather view of
// them (gp_build_fallback_view, one CTA per instance group).  on_device: the orders are device arrays
// (gp_prepare_cluster_zones' held orders) and are read in place.
static gp_status stage_fallback_view(gp_ctx* c, const gp_instance_groups& ig, bool on_device, cudaStream_t st, GatherSlots* fb) {
    const int32_t G = ig.n_instance_groups;
    const size_t ne = (size_t)ig.exec_off[G], nd = (size_t)ig.drv_off[G];
    const size_t n_off = G == 1 ? 0 : (size_t)G + 1;          // one instance group: the whole orders, no offsets
    Arena ar{c->fbview, st};
    const auto eord = ar.take<int32_t>(on_device ? 0 : ne), dord = ar.take<int32_t>(on_device ? 0 : nd),
               npos = ar.take<int32_t>((size_t)c->n_nodes), fbe = ar.take<int32_t>(ne), fbd = ar.take<int32_t>(nd), fbp = ar.take<int32_t>(nd);
    const auto eoff = ar.take<int32_t>(n_off), doff = ar.take<int32_t>(n_off);
    ar.reserve();
    if (!on_device) {
        ar.put(eord, ig.exec_order);
        ar.put(dord, ig.drv_order);
    }
    const int32_t* d_eoff = n_off ? ar.put(eoff, ig.exec_off) : nullptr;
    const int32_t* d_doff = n_off ? ar.put(doff, ig.drv_off) : nullptr;
    GP_TRY(ar.check(c));
    gp_build_fallback_view<<<(unsigned)G, 1024, 0, st>>>((int32_t)ne, (int32_t)nd, d_eoff, d_doff, on_device ? ig.exec_order : ar.ptr(eord),
                                                         on_device ? ig.drv_order : ar.ptr(dord), c->node_slot.as<int32_t>(), ar.ptr(npos),
                                                         ar.ptr(fbe), ar.ptr(fbd), ar.ptr(fbp));
    c->last.kernel_launches += 1;
    *fb = GatherSlots{ar.ptr(fbe), ar.ptr(fbd), ar.ptr(fbp), (int32_t)ne, (int32_t)nd};
    return GP_OK;
}

// zone / driver / ExecutorNodes (T entries) / averages to the host, one synchronise, then the kernels' validation errors
static gp_status finish_zone_results(gp_ctx* c, Arena& ar, gp_zone_results* out, Piece<int32_t> zone, Piece<int32_t> drv,
                                     Piece<int32_t> exe, Piece<double> avg, size_t T) {
    ar.get(out->zone, zone);
    ar.get(out->driver_node, drv);
    ar.get(out->executor_nodes, exe.part(0, T));
    ar.get(out->avg_efficiency, avg);
    GP_TRY(ar.sync(c));
    return host_error(c);
}

// Independent zone packs of a batch, shared by gp_pack_batch_zones (the zones are every instance group, no fallback) and
// gp_pack_batch_az_aware (zones 0..Z-1 with tightly-pack, plus the undivided orders `az` of the fallback, already
// validated; az_dev: they are device arrays).  Argument checks common to both are here.
static gp_status batch_zones_run(gp_ctx* c, const gp_apps* a, gp_algo algo, int32_t Z, const gp_az_orders* az, bool az_dev,
                                 gp_zone_results* out, const char* who) {
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, who, "missing app/result arrays");
    if ((int64_t)Q * Z > 0x7fffffffLL) return fail(c, GP_ERR_INVALID, who, "n_apps x zones too large");
    const int64_t* off = a->exec_out_off;
    if (!off) {
        c->host_off.resize((size_t)Q + 1);
        int64_t acc = 0;
        for (int32_t i = 0; i < Q; ++i) { c->host_off[(size_t)i] = acc; acc += a->exe_count[i] > 0 ? a->exe_count[i] : 0; }
        c->host_off[(size_t)Q] = acc;
        off = c->host_off.data();
    }
    const int64_t total = off[Q];
    if (total < 0 || total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, who, "executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, who, "executor_nodes is NULL");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, R = q * (size_t)Z, T = (size_t)total;
    Arena ar{c->zonebuf, st};
    const auto in = ar.take<int64_t>(6 * q);
    const auto cnt = ar.take<int32_t>(q);
    const auto off_p = ar.take<int64_t>(q + 1), rows = ar.take<int64_t>(6 * R);
    const auto rcnt = ar.take<int32_t>(R), rgrp = ar.take<int32_t>(R);
    const auto roff = ar.take<int64_t>(R + 1);
    const auto rdrv = ar.take<int32_t>(R), rexe = ar.take<int32_t>((size_t)Z * T + 1), zone = ar.take<int32_t>(q), drv = ar.take<int32_t>(q),
               exe = ar.take<int32_t>(T + 1);
    const auto avg = ar.take<double>(4 * q);
    // az-aware: the fallback's PrepApp records and list
    const size_t QF = az ? q : 0;
    const auto prep = ar.take<PrepApp>(QF);
    const auto list = ar.take<int32_t>(QF);
    ar.reserve();
    const SixCols six = upload_app_columns(ar, a, off, in, cnt, off_p);
    GP_TRY(ar.check(c));
    const int TH = 256;
    // the efficiencies read the availability in node-table order: refresh that copy from the slots (a FIFO batch may
    // have charged them since gp_set_snapshot)
    if (c->n_slots > 0)
        gp_scatter_slots<<<(c->n_slots + TH - 1) / TH, TH, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(), c->slot_node.as<int32_t>(),
                                                                   c->node_cpu.as<int64_t>(), c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
    gp_zone_expand<<<(unsigned)((R + 1 + TH - 1) / TH), TH, 0, st>>>(Q, Z, six, ar.ptr(cnt), ar.ptr(off_p), ar.ptr(rows), ar.ptr(rcnt),
                                                                      ar.ptr(rgrp), ar.ptr(roff));
    int2* scratch = nullptr;
    GP_TRY(pack_begin(c, (int32_t)R, algo, GP_MODE_INDEPENDENT, (int64_t)Z * total, false, &scratch, st));
    DevApps dv{};
    for (int k = 0; k < 6; ++k) dv.cols.q[k] = ar.ptr(rows) + R * (size_t)k;
    dv.cols.count = ar.ptr(rcnt); dv.cols.group = ar.ptr(rgrp); dv.cols.off = ar.ptr(roff);
    dv.cols.bits = 64; dv.cols.mem_shift = 0; dv.skip = nullptr; dv.n = (int32_t)R;
    DevResults dr{ar.ptr(rdrv), ar.ptr(rexe), (int64_t)Z * total, 32};
    GP_TRY(pack_device_range(c, dv, 0, (int32_t)R, 0, algo, GP_MODE_INDEPENDENT, dr, scratch, st, 0));
    c->ev_chunks = 1;
    ZoneChooseIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.avail[0] = c->node_cpu.as<long long>(); zi.avail[1] = c->node_mem.as<long long>(); zi.avail[2] = c->node_gpu.as<long long>();
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    for (int k = 0; k < 3; ++k) { zi.drv[k] = six.p[k]; zi.exe[k] = six.p[3 + k]; }
    zi.count = ar.ptr(cnt); zi.out_off = ar.ptr(off_p);
    zi.row_driver = ar.ptr(rdrv); zi.row_exec = ar.ptr(rexe);
    zi.n_apps = Q; zi.n_zones = Z; zi.executors_reserved = algo == GP_TIGHTLY_PACK ? 1 : 0;
    gp_zone_choose<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(zi, ar.ptr(zone), ar.ptr(drv), ar.ptr(exe),
                                                                       out->avg_efficiency ? ar.ptr(avg) : nullptr);
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    if (az) {
        // the applications no zone won: SparkBinPack(tightlyPackExecutors) over the undivided orders, still on the device
        // (az_aware_pack_tightly.go:33-37).  The list length and the fallback's claim counter are zeroed by pack_begin;
        // stats [2..3] restart so that scan_path_apps / _nodes count the fallback alone.
        DevStatus* ds = c->status();
        unsigned long long* d_stats = ds->head.stats;
        GP_CUDA(c, cudaMemsetAsync(d_stats + 2, 0, 16, st));
        int32_t* listed = ar.ptr(list);
        gp_az_fallback_list<<<(unsigned)((q + TH - 1) / TH), TH, 0, st>>>(Q, ar.ptr(zone), listed, &ds->az_listed);
        AppColumns cols{};
        for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
        cols.count = ar.ptr(cnt); cols.group = nullptr; cols.off = ar.ptr(off_p); cols.bits = 64; cols.mem_shift = 0;
        gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
            Q, cols, nullptr, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, ar.ptr(prep), &ds->head.err, &c->host_status()->err_word);
        GatherSlots fb;
        const OneInstanceGroup one(c->n_groups, az);
        GP_TRY(stage_fallback_view(c, one.ig, az_dev, st, &fb));
        int& per_sm = c->az_fallback_ctas_per_sm;
        if (per_sm == 0) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_pack_az_fallback, kAzFallbackThreads, 0);
            if (per_sm < 1) per_sm = 1;
        }
        int64_t blocks = ((int64_t)Q * 32 + kAzFallbackThreads - 1) / kAzFallbackThreads;   // the list holds at most Q
        if (blocks > (int64_t)c->sm_count * per_sm) blocks = (int64_t)c->sm_count * per_sm;
        gp_pack_az_fallback<<<(unsigned)blocks, kAzFallbackThreads, 0, st>>>(make_snapshot(c), ar.ptr(prep), listed, &ds->az_listed, fb, ar.ptr(drv),
                                                                            ar.ptr(exe), d_stats, &ds->az_claim);
        GP_CUDA(c, cudaGetLastError());
        c->last.kernel_launches += 3;
    }
    return finish_zone_results(c, ar, out, zone, drv, exe, avg, T);
}

gp_status gp_pack_batch_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_zone_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), c->held.full_sched(), "gp_pack_batch_zones"));
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: the single-AZ packers are tightly-pack and minimal-fragmentation (single_az_pack_tightly.go, single_az_minimal_fragmentation.go)");
    GP_TRY(require(c, c->held.one_instance_group(), "gp_pack_batch_zones"));
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

// The undivided orders of az-aware-tightly-pack against the snapshot gp_set_snapshot laid out, in O(N): every entry of
// instance group b's orders a node of b's groups in that role, every node once over all instance groups (so b's orders are
// a permutation of b's nodes in that role); every zone group's order = its instance group's undivided order restricted to
// that group's nodes (the fallback and the zone packs must see the same priorities).  ig.group_off and ig.n_zones are
// already checked; ig.exec_off / ig.drv_off are present.
static gp_status check_az_orders(gp_ctx* c, const gp_instance_groups& ig, const char* who) {
    GP_TRY(require(c, c->held.host_copy(false), who));
    const std::string w(who);
    const int32_t G = ig.n_instance_groups;
    if (ig.exec_off[G] != c->n_exec || ig.drv_off[G] != c->n_drv)
        return fail(c, GP_ERR_INVALID, w + ": order lengths must equal the snapshot's exec_off[n_groups] / drv_off[n_groups]");
    for (int32_t b = 0; b < G; ++b)
        if (ig.exec_off[0] != 0 || ig.drv_off[0] != 0 || ig.exec_off[b + 1] < ig.exec_off[b] || ig.drv_off[b + 1] < ig.drv_off[b])
            return fail(c, GP_ERR_INVALID, w + ": exec_off / drv_off must be monotone from 0");
    if ((c->n_exec > 0 && !ig.exec_order) || (c->n_drv > 0 && !ig.drv_order))
        return fail(c, GP_ERR_INVALID, w + ": order arrays missing");
    const uint32_t N = (uint32_t)c->n_nodes;
    const int32_t* owner = c->v_owner.data();
    const int32_t* pos = c->v_pos.data();
    for (int role = 0; role < 2; ++role) {
        const int32_t* off = role == 0 ? ig.exec_off : ig.drv_off;
        const int32_t* ord = role == 0 ? ig.exec_order : ig.drv_order;
        const char* name = role == 0 ? "exec_order" : "drv_order";
        std::vector<uint8_t>& seen = role == 0 ? c->v_seen_e : c->v_seen_d;
        seen.assign((size_t)N, 0);
        std::vector<int32_t>& next = c->v_zone_next;     // next expected position in each zone group's order
        next.assign((size_t)c->n_groups, 0);
        for (int32_t b = 0; b < G; ++b) {
            const int32_t g_lo = ig.group_off[b], g_hi = ig.group_off[b + 1], z_hi = g_lo + ig.n_zones[b];
            for (int32_t i = off[b]; i < off[b + 1]; ++i) {
                const uint32_t v = (uint32_t)ord[i];
                if (v >= N) return fail(c, GP_ERR_INVALID, w + ": " + name + " entry out of range");
                if (seen[v]) return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node twice");
                seen[v] = 1;
                const int32_t ow = owner[v];
                if (ow < 0 || !(ow & (1 << role)))
                    return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node the snapshot does not list as " +
                                                       (role == 0 ? "an executor" : "a driver") + " candidate");
                const int32_t g = ow >> 2;
                if (g < g_lo || g >= g_hi)
                    return fail(c, GP_ERR_INVALID, w + ": " + name + " of instance group " + std::to_string(b) +
                                                       " lists a node of another instance group");
                if (g < z_hi && pos[(size_t)role * N + v] != next[(size_t)g]++)
                    return fail(c, GP_ERR_INVALID, w + ": zone group " + std::to_string(g) + "'s " +
                                                       (role == 0 ? "executor" : "driver") + " order is not " + name + " restricted to its nodes");
            }
        }
    }
    return GP_OK;
}

// The az-aware entries' NULL arguments.  orders == NULL stands for the undivided orders and n_zones gp_prepare_cluster_zones
// (GP_LAYOUT_AZ_AWARE) left on the device -- *o then points at them; after any other snapshot it is refused.
static gp_status held_az_orders(gp_ctx* c, const gp_apps* a, const gp_zone_results* out, const gp_az_orders** o, const char* who) {
    if (!*o) GP_TRY(require(c, c->held.az_orders(), who));
    if (!*o) *o = c->held.orders();
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, who, "NULL apps/orders/results");
    return GP_OK;
}

}  // extern "C"

gp_status zone_fifo_kind(gp_ctx* c, gp_binpacker packer, gp_mode mode, const char* who, int* kind) {
    if (packer == GP_BP_SINGLE_AZ_TIGHTLY_PACK) *kind = GP_TIGHTLY_PACK;
    else if (packer == GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION) *kind = GP_MINIMAL_FRAGMENTATION;
    else if (packer == GP_BP_AZ_AWARE_TIGHTLY_PACK) *kind = kZoneAzAware;
    else return fail(c, GP_ERR_INVALID, who, "packer must be GP_BP_SINGLE_AZ_TIGHTLY_PACK, GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION or "
                                             "GP_BP_AZ_AWARE_TIGHTLY_PACK");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, who, "mode must be one of the FIFO modes");
    return require(c, c->held.full_sched(), who);
}

// The FIFO loop over zones in one launch (gangpack_zonefifo.cuh), one CTA per instance group of `ig` (already validated),
// shared by gp_pack_fifo_zones (kind = 0 tightly-pack, 2 minimal-fragmentation; one instance group whose zones are every
// snapshot group), gp_pack_fifo_az_aware (kind = kZoneAzAware; one instance group, zones 0..n_zones-1, plus the undivided
// orders of the fallback; az_dev: they are device arrays), gp_pack_fifo_zones_groups (either, per instance group) and
// gp_pack_fifo_zones_groups_driver_table (its columns on the device).  c->zone_groups holds, per instance group, its
// application count in q_end and its largest exe_count in row_pitch; total = the ExecutorNodes entries.
gp_status fifo_zones_body(gp_ctx* c, int32_t Q, int64_t total, const ZoneFifoApps& src, int kind, gp_mode mode,
                          const gp_instance_groups& ig, bool az_dev, gp_zone_results* out, const char* who) {
    const bool azk = kind == kZoneAzAware;
    const int32_t G = ig.n_instance_groups;
    const gp_apps* a = src.host;
    std::vector<ZoneFifoGroup>& grp = c->zone_groups;
    if (total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, who, "executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, who, "executor_nodes is NULL");
    // per instance group: its zones, its queue range and its scratch rows (n_zones, az-aware: + the fallback row)
    int32_t qb = 0;
    int64_t rows = 0;
    for (int32_t b = 0; b < G; ++b) {
        ZoneFifoGroup& g = grp[(size_t)b];
        g.zone0 = ig.group_off[b];
        g.n_zones = azk ? ig.n_zones[b] : ig.group_off[b + 1] - ig.group_off[b];
        const int32_t n = g.q_end;
        g.q_begin = g.q_end = qb;                          // q_end: the cursor of the fill below
        qb += n;
        g.row_pitch = (std::max<int64_t>(g.row_pitch, 1) + 3) & ~(int64_t)3;
        g.row_base = rows;
        rows += (int64_t)(g.n_zones + (azk ? 1 : 0)) * g.row_pitch;
        if (azk) {
            g.e0 = ig.exec_off[b]; g.ne = ig.exec_off[b + 1] - g.e0;
            g.d0 = ig.drv_off[b]; g.nd = ig.drv_off[b + 1] - g.d0;
        }
    }
    std::vector<int32_t>& queue = c->zone_queue;
    if (a) {                                                // stable counting sort of the applications by instance group
        queue.resize((size_t)Q);
        for (int32_t i = 0; i < Q; ++i) queue[(size_t)grp[(size_t)(src.group ? src.group[i] : 0)].q_end++] = i;
    } else {                                                // device columns: already in instance-group order (src.queue)
        for (int32_t b = 0; b < G; ++b) grp[(size_t)b].q_end = b + 1 < G ? grp[(size_t)b + 1].q_begin : qb;
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)total, RP = (size_t)rows, qh = a ? q : 0;
    Arena ar{c->zonebuf, st};
    const auto in = ar.take<int64_t>(6 * qh);
    const auto cnt = ar.take<int32_t>(qh);
    const auto off_p = ar.take<int64_t>(a ? q + 1 : 0);
    const auto skip = ar.take<uint8_t>(qh);
    const auto gdesc = ar.take<ZoneFifoGroup>((size_t)G);
    const auto qidx = ar.take<int32_t>(qh);
    const auto rexe = ar.take<int32_t>(RP);
    const auto rlist = ar.take<int2>(kind == GP_MINIMAL_FRAGMENTATION ? RP : 0);
    const auto zone = ar.take<int32_t>(q), drv = ar.take<int32_t>(q), exe = ar.take<int32_t>(T + 1);
    const auto avg_p = ar.take<double>(4 * q);
    ar.reserve();
    GP_TRY(ar.check(c));
    int2* unused = nullptr;
    GP_TRY(pack_begin(c, Q, GP_TIGHTLY_PACK, mode, total, false, &unused, st));
    AppColumns cols{};
    SixCols six{};
    for (int k = 0; k < 6; ++k) six.p[k] = src.q[k];
    const int32_t* d_cnt = src.count;
    const int64_t* d_off = src.off;
    const uint8_t* d_skip = src.skip;
    const int32_t* d_queue = src.queue;
    if (a) {
        six = upload_app_columns(ar, a, src.off, in, cnt, off_p);
        d_cnt = ar.ptr(cnt); d_off = ar.ptr(off_p);
        d_skip = ar.put(skip, a->skip_if_no_fit);
        d_queue = ar.put(qidx, queue.data());
    }
    ar.put(gdesc, grp.data());
    GP_TRY(ar.check(c));
    for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
    cols.count = d_cnt; cols.group = nullptr; cols.off = d_off; cols.bits = 64; cols.mem_shift = 0;
    DevStatus* ds = c->status();
    unsigned long long* d_stats = ds->head.stats;
    PrepApp* prep = c->prep.as<PrepApp>();
    gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
        Q, cols, d_skip, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, prep, &ds->head.err, &c->host_status()->err_word);
    Snapshot snap = make_snapshot(c);
    ZoneFifoIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    zi.node_slot = c->node_slot.as<int32_t>();
    zi.row_exec = ar.ptr(rexe);
    zi.row_list = kind == GP_MINIMAL_FRAGMENTATION ? ar.ptr(rlist) : nullptr;
    zi.groups = ar.ptr(gdesc); zi.queue = d_queue;
    double* avg = out->avg_efficiency ? ar.ptr(avg_p) : nullptr;
    int32_t* zo = ar.ptr(zone); int32_t* dq = ar.ptr(drv); int32_t* eo = ar.ptr(exe);
    GatherSlots fb{};
    if (azk) GP_TRY(stage_fallback_view(c, ig, az_dev, st, &fb));
    const unsigned ctas = (unsigned)G;                 // one per instance group
    if (kind == GP_TIGHTLY_PACK) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<0, 1><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<0, 2><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else if (kind == GP_MINIMAL_FRAGMENTATION) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<2, 1><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<2, 2><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<kZoneAzAware, 1><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
        else gp_pack_fifo_zones_cta<kZoneAzAware, 2><<<ctas, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
    }
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    GP_TRY(refresh_views(c, st));                       // the compact view follows the charged slots
    return finish_zone_results(c, ar, out, zone, drv, exe, avg_p, T);
}

extern "C" {

// fifo_zones_body over host columns.  group: the instance group of every application, NULL = 0.  Argument checks common to
// gp_pack_fifo_zones, gp_pack_fifo_az_aware and gp_pack_fifo_zones_groups are here.
static gp_status fifo_zones_run(gp_ctx* c, const gp_apps* a, const int32_t* group, int kind, gp_mode mode, const gp_instance_groups& ig,
                                bool az_dev, gp_zone_results* out, const char* who) {
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, who, "missing app/result arrays");
    const int32_t G = ig.n_instance_groups;
    // one pass over the queue: ExecutorNodes offsets, and per instance group its application count (in q_end) and its
    // largest exe_count (in row_pitch)
    std::vector<ZoneFifoGroup>& grp = c->zone_groups;
    grp.assign((size_t)G, ZoneFifoGroup{});
    std::vector<int64_t>& hoff = c->host_off;
    hoff.resize((size_t)Q + 1);
    int64_t acc = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        hoff[(size_t)i] = acc; acc += k;
        const int32_t b = group ? group[i] : 0;
        if (b < 0 || b >= G) return fail(c, GP_ERR_INVALID, who, "an application's group is outside [0, n_instance_groups)");
        ZoneFifoGroup& g = grp[(size_t)b];
        ++g.q_end;
        if (k > g.row_pitch) g.row_pitch = k;
    }
    hoff[(size_t)Q] = acc;
    if (a->exec_out_off)
        for (int32_t i = 0; i <= Q; ++i)
            if (a->exec_out_off[i] != hoff[(size_t)i]) return fail(c, GP_ERR_INVALID, who, "exec_out_off must be the prefix sum of exe_count (or NULL)");
    ZoneFifoApps src{};
    src.host = a; src.group = group; src.off = hoff.data();
    return fifo_zones_body(c, Q, acc, src, kind, mode, ig, az_dev, out, who);
}

// the FIFO loop with a single-AZ packer in one launch
gp_status gp_pack_fifo_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_mode mode, gp_zone_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), c->held.full_sched(), "gp_pack_fifo_zones"));
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: the single-AZ packers are tightly-pack and minimal-fragmentation");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones)");
    GP_TRY(require(c, c->held.one_instance_group(), "gp_pack_fifo_zones"));
    if (c->n_groups > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: more than 64 zones");
    const OneInstanceGroup one(c->n_groups, nullptr);
    return fifo_zones_run(c, a, nullptr, (int)algo, mode, one.ig, false, out, "gp_pack_fifo_zones");
}

// the FIFO loop with az-aware-tightly-pack in one launch: the zone packs plus the undivided fallback on the device
gp_status gp_pack_fifo_az_aware(gp_ctx* c, const gp_apps* a, gp_mode mode, const gp_az_orders* o, gp_zone_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), "gp_pack_fifo_az_aware"));
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones, "
                                       "then gp_pack_batch over the undivided orders)");
    GP_TRY(require(c, c->held.full_sched(), "gp_pack_fifo_az_aware"));
    GP_TRY(held_az_orders(c, a, out, &o, "gp_pack_fifo_az_aware"));
    const bool held = o == c->held.orders();
    const int32_t Z = o->n_zones;
    if (Z < 0 || Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones must be 0..64");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones exceeds the snapshot's instance groups");
    const OneInstanceGroup one(c->n_groups, o);
    if (!held) GP_TRY(check_az_orders(c, one.ig, "gp_pack_fifo_az_aware"));
    return fifo_zones_run(c, a, nullptr, kZoneAzAware, mode, one.ig, held, out, "gp_pack_fifo_az_aware");
}

}  // extern "C"

// gp_pack_fifo_zones_groups(groups == NULL): the layout gp_prepare_cluster_zones_groups left, from its host words and its
// device orders (built by the library: no order check)
gp_status held_groups_layout(gp_ctx* c, int kind, const char* who, gp_instance_groups* held) {
    const bool azk = kind == kZoneAzAware;
    GP_TRY(require(c, c->held.groups_layout(azk), who));
    *held = c->held.groups();
    for (int32_t b = 0; b < held->n_instance_groups; ++b)
        if ((azk ? held->n_zones[b] : held->group_off[b + 1] - held->group_off[b]) > kZoneFifoMaxZones)
            return fail(c, GP_ERR_INVALID, who, "more than 64 candidate zones in an instance group");
    return GP_OK;
}

extern "C" {

static gp_status held_groups_run(gp_ctx* c, const gp_apps* a, int kind, gp_mode mode, gp_zone_results* out, const char* who) {
    gp_instance_groups held{};
    GP_TRY(held_groups_layout(c, kind, who, &held));
    return fifo_zones_run(c, a, a->group, kind, mode, held, kind == kZoneAzAware, out, who);
}

// the FIFO loop of every instance group with a zone-aware packer, one CTA per instance group, in one launch
gp_status gp_pack_fifo_zones_groups(gp_ctx* c, const gp_apps* a, gp_binpacker packer, gp_mode mode, const gp_instance_groups* ig,
                                    gp_zone_results* out) {
    const char* who = "gp_pack_fifo_zones_groups";
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), who));
    int kind;
    GP_TRY(zone_fifo_kind(c, packer, mode, who, &kind));
    if (!ig) {
        if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, who, "NULL apps/results");
        return held_groups_run(c, a, kind, mode, out, who);
    }
    GP_TRY(require(c, c->held.host_copy(true), who));
    if (!a || !out || !ig || a->n_apps < 0) return fail(c, GP_ERR_INVALID, who, "NULL apps/groups/results");
    const int32_t G = ig->n_instance_groups;
    const int32_t* goff = ig->group_off;
    if (G < 0 || !goff) return fail(c, GP_ERR_INVALID, who, "n_instance_groups is negative or group_off is NULL");
    if (goff[0] != 0 || goff[G] != c->n_groups) return fail(c, GP_ERR_INVALID, who, "group_off must run from 0 to the snapshot's n_groups");
    const bool azk = kind == kZoneAzAware;
    if (azk && (!ig->n_zones || !ig->exec_off || !ig->drv_off))
        return fail(c, GP_ERR_INVALID, who, "az-aware-tightly-pack needs n_zones, exec_off and drv_off");
    for (int32_t b = 0; b < G; ++b) {
        const int64_t n = (int64_t)goff[b + 1] - goff[b];
        if (n < 0) return fail(c, GP_ERR_INVALID, who, "group_off is not monotone");
        const int64_t Z = azk ? ig->n_zones[b] : n;
        if (Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, who, "more than 64 candidate zones in an instance group");
        if (Z < 0 || Z > n) return fail(c, GP_ERR_INVALID, who, "n_zones[i] must be 0 .. the number of groups of instance group i");
    }
    if (azk) GP_TRY(check_az_orders(c, *ig, who));
    return fifo_zones_run(c, a, a->group, kind, mode, *ig, false, out, who);
}

// az-aware-tightly-pack for a batch of independent decisions: the zone packs, the zone choice and the undivided fallback
// on the device, one stream synchronise
gp_status gp_pack_batch_az_aware(gp_ctx* c, const gp_apps* a, const gp_az_orders* o, gp_zone_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), c->held.full_sched(), "gp_pack_batch_az_aware"));
    GP_TRY(held_az_orders(c, a, out, &o, "gp_pack_batch_az_aware"));
    const bool held = o == c->held.orders();
    const int32_t Z = o->n_zones;
    if (Z < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones is negative");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones exceeds the snapshot's instance groups");
    const OneInstanceGroup one(c->n_groups, o);
    if (!held) GP_TRY(check_az_orders(c, one.ig, "gp_pack_batch_az_aware"));
    return batch_zones_run(c, a, GP_TIGHTLY_PACK, Z, o, held, out, "gp_pack_batch_az_aware");
}

gp_status gp_reserve_placements(gp_ctx* c, const gp_apps* a, const gp_results* placed, int32_t subtract, gp_reservation_table* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), "gp_reserve_placements"));
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
    Arena ar{c->zonebuf, st};
    const auto in = ar.take<int64_t>(6 * q);
    const auto cnt = ar.take<int32_t>(q);
    const auto off_p = ar.take<int64_t>(q + 1), roff_p = ar.take<int64_t>(q + 1);
    const auto drv = ar.take<int32_t>(q), exe = ar.take<int32_t>(T + 1), ra = ar.take<int32_t>(R + 1), rs = ar.take<int32_t>(R + 1),
               rn = ar.take<int32_t>(R + 1);
    const auto rc = ar.take<long long>(R + 1), rm = ar.take<long long>(R + 1), rg = ar.take<long long>(R + 1);
    ar.reserve();
    ReserveIn ri{};
    ri.cols = upload_app_columns(ar, a, off.data(), in, cnt, off_p);
    ri.row_off = ar.put(roff_p, roff);
    ri.driver = ar.put(drv, placed->driver_node);
    ar.put(exe.part(0, T), placed->executor_nodes);
    GP_TRY(ar.check(c));
    ri.count = ar.ptr(cnt); ri.off = ar.ptr(off_p); ri.exec = ar.ptr(exe); ri.n_apps = Q; ri.subtract = subtract ? 1 : 0;
    ReserveOut ro{ar.ptr(ra), ar.ptr(rs), ar.ptr(rn), ar.ptr(rc), ar.ptr(rm), ar.ptr(rg)};
    const int TH = 256;
    gp_reserve_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, ro, c->node_slot.as<int32_t>(), c->pair.as<longlong2>(), c->sgpu.as<long long>(),
                                                                        c->node_cpu.as<long long>(), c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    if (subtract) GP_TRY(refresh_views(c, st));
    if (out) {
        ar.get(out->app, ra.part(0, R));
        ar.get(out->slot, rs.part(0, R));
        ar.get(out->node, rn.part(0, R));
        ar.get(out->cpu_milli, rc.part(0, R));
        ar.get(out->mem_bytes, rm.part(0, R));
        ar.get(out->gpu, rg.part(0, R));
    }
    GP_TRY(ar.sync(c));
    if (out) out->n_rows = rows;
    return GP_OK;
}

gp_status gp_apply_usage_delta(gp_ctx* c, int64_t n_rows, const int32_t* node, const int64_t* cpu, const int64_t* mem, const int64_t* gpu, int32_t sign) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot(), "gp_apply_usage_delta"));
    if (n_rows < 0 || (sign != 1 && sign != -1) || (n_rows > 0 && (!node || !cpu || !mem))) return fail(c, GP_ERR_INVALID, "gp_apply_usage_delta: bad arguments");
    if (n_rows == 0) return GP_OK;
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t v[3] = {cpu[r], mem[r], gpu ? gpu[r] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_apply_usage_delta: |quantity| >= 2^61");
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t R = (size_t)n_rows;
    Arena ar{c->zonebuf, st};
    const auto cp = ar.take<long long>(R), mp = ar.take<long long>(R), gp = ar.take<long long>(R);
    const auto np = ar.take<int32_t>(R);
    ar.reserve();
    const long long* d_cpu = ar.put(cp, cpu);
    const long long* d_mem = ar.put(mp, mem);
    const long long* d_gpu = ar.put(gp, gpu);
    const int32_t* d_node = ar.put(np, node);
    GP_TRY(ar.check(c));
    const int TH = 256;
    gp_usage_delta<<<(unsigned)((R + TH - 1) / TH), TH, 0, st>>>(n_rows, d_node, d_cpu, d_mem, d_gpu, sign, c->n_nodes, c->node_slot.as<int32_t>(),
                                                                  c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_cpu.as<long long>(),
                                                                  c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    GP_TRY(refresh_views(c, st));
    return ar.sync(c);
}

// ---- computeAvgPackingEfficiencyForResult over the whole node table, exactly summed (gangpack_efficiency.cuh) ----------
// The efficiency kernels' status word (kEffErr* bits)
static const Refusal kEffRefusals[] = {
    {kEffErrQuantity, GP_ERR_UNREPRESENTABLE, "a per-node reserved amount is >= 2^61"},
    {kEffErrRange, GP_ERR_UNREPRESENTABLE, "an efficiency term outside the exact accumulator's range"},
};

}  // extern "C"

// gp_packing_efficiency (ig NULL: every node of the table, one segment) and gp_packing_efficiency_groups (row i over the nodes
// v with ig[v] == a->group[i]): the host pass over the rows, the (segmented) base pass and the row pass.
static gp_status packing_efficiency(gp_ctx* c, const gp_apps* a, gp_algo algo, const gp_results* placed, gp_mode charged, const int32_t* ig,
                                    int32_t n_ig, double* avg_out, const char* who) {
    GP_TRY(require(c, c->held.snapshot("no snapshot (gp_set_snapshot, gp_prepare_cluster or gp_prepare_cluster_zones first)"),
                   c->held.efficiency_sched(), who));
    if (!a || !placed || a->n_apps < 0) return fail(c, GP_ERR_INVALID, who, "NULL apps/placed");
    if (algo != GP_TIGHTLY_PACK && algo != GP_DISTRIBUTE_EVENLY && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, who, "unknown algo");
    if (charged != GP_MODE_INDEPENDENT && charged != GP_MODE_FIFO_REFERENCE && charged != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, who, "unknown charged mode");
    if (!ig && charged != GP_MODE_INDEPENDENT && a->n_apps != 1)
        return fail(c, GP_ERR_INVALID, who, "a FIFO charged mode adds back ONE application's usage: n_apps must be 1");
    const int32_t Q = a->n_apps, N32 = c->n_nodes;
    // instance groups: the nodes bucketed by instance group (stable counting sort), seg[0 .. G] their CSR offsets
    std::vector<int32_t>& seg = c->eff_seg;
    if (ig) {
        if (n_ig < 1) return fail(c, GP_ERR_INVALID, who, "n_instance_groups must be >= 1");
        seg.assign((size_t)n_ig + 1, 0);
        for (int32_t v = 0; v < N32; ++v) {
            if (ig[v] < -1 || ig[v] >= n_ig) return fail(c, GP_ERR_INVALID, who, "instance_group outside [-1, n_instance_groups)");
            if (ig[v] >= 0) ++seg[(size_t)ig[v] + 1];
        }
        for (int32_t g = 0; g < n_ig; ++g) seg[(size_t)g + 1] += seg[(size_t)g];
        for (int32_t i = 0; i < Q; ++i) {
            const int32_t g = a->group ? a->group[i] : 0;
            if (g < 0 || g >= n_ig) return fail(c, GP_ERR_INVALID, who, "apps->group outside [0, n_instance_groups)");
        }
        if (charged != GP_MODE_INDEPENDENT) {           // each row adds back usage on its own instance group's nodes only
            std::vector<uint8_t>& seen = c->v_seen_e;
            seen.assign((size_t)n_ig, 0);
            for (int32_t i = 0; i < Q; ++i) {
                const int32_t g = a->group ? a->group[i] : 0;
                if (seen[(size_t)g]) return fail(c, GP_ERR_INVALID, who, "a FIFO charged mode adds back ONE application's usage per instance group: two rows name one instance group");
                seen[(size_t)g] = 1;
            }
        }
    }
    if (Q == 0) return GP_OK;
    if (!avg_out || !a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !placed->driver_node)
        return fail(c, GP_ERR_INVALID, who, "missing app/result arrays");
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
        if (d >= N32) return fail(c, GP_ERR_INVALID, who, "driver_node out of range");
        if (d < 0) continue;
        const int32_t g = ig && a->group ? a->group[i] : 0;
        if (ig && ig[d] != g) return fail(c, GP_ERR_INVALID, who, "driver_node outside the application's instance group");
        for (const int64_t* col : qc) {
            if (!col) continue;
            if (col[i] < 0) return fail(c, GP_ERR_INVALID, who, "negative request");
            if (col[i] >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, who, "request >= 2^61");
        }
        if (k > 0 && !placed->executor_nodes) return fail(c, GP_ERR_INVALID, who, "executor_nodes is NULL");
        if (off[(size_t)i] < 0 || off[(size_t)i] + k > placed->executor_nodes_cap)
            return fail(c, GP_ERR_CAPACITY, who, "offsets exceed executor_nodes_cap");
        for (int64_t t = 0; t < k; ++t) {
            const int32_t n = placed->executor_nodes[off[(size_t)i] + t];
            if (n < 0 || n >= N32) return fail(c, GP_ERR_INVALID, who, "executor node out of range");
            if (ig && ig[n] != g) return fail(c, GP_ERR_INVALID, who, "executor node outside the application's instance group");
        }
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    const int64_t total = placed->executor_nodes_cap < off[(size_t)Q] ? placed->executor_nodes_cap : off[(size_t)Q];
    const size_t G = ig ? (size_t)n_ig : 1, NS = ig ? (size_t)seg[G] : 0;
    if (ig) {                                           // bucket the nodes: seg[G + 1 ..] = the nodes of each instance group
        seg.resize(G + 1 + NS);
        std::vector<int32_t> cur(seg.begin(), seg.begin() + (ptrdiff_t)G);      // next free position of each bucket
        for (int32_t v = 0; v < N32; ++v)
            if (ig[v] >= 0) seg[G + 1 + (size_t)cur[(size_t)ig[v]]++] = v;
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)(total > 0 ? total : 0), N = (size_t)N32;
    const int TH = kEffThreads;
    // CTAs per segment: up to four per SM over all segments together, at most one per 256 nodes of the largest segment
    size_t longest = ig ? 0 : N;
    for (size_t g = 0; ig && g < G; ++g) longest = std::max<size_t>(longest, (size_t)(seg[g + 1] - seg[g]));
    const size_t per_seg = ((size_t)c->sm_count * 4 + G - 1) / G;
    const int n_part = (int)std::max<size_t>(1, std::min<size_t>((longest + TH - 1) / TH, per_seg));
    Arena ar{c->zonebuf, st};
    const auto in = ar.take<int64_t>(6 * q);
    const auto cnt = ar.take<int32_t>(q);
    const auto off_p = ar.take<int64_t>(q + 1);
    const auto drv = ar.take<int32_t>(q), exe = ar.take<int32_t>(T + 1);
    const auto part = ar.take<EffAcc>((size_t)n_part * G), base = ar.take<EffAcc>(G);
    const auto avg = ar.take<double>(4 * q);
    const auto err = ar.take<int>(1);
    const auto segp = ar.take<int32_t>(ig ? G + 1 + NS : 0), grp = ar.take<int32_t>(ig && a->group ? q : 0);
    ar.reserve();
    EffRowsIn ri{};
    ri.cols = upload_app_columns(ar, a, off.data(), in, cnt, off_p);
    ri.driver = ar.put(drv, placed->driver_node);
    ar.put(exe.part(0, T), placed->executor_nodes);
    int* d_err = ar.zero(err);
    const int32_t* d_seg = ig ? ar.put(segp, seg.data()) : nullptr;
    ri.group = ig ? ar.put(grp, a->group) : nullptr;
    GP_TRY(ar.check(c));
    EffBaseIn bi{};
    bi.av = SnapshotAvail{c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_slot.as<int32_t>(), c->node_cpu.as<long long>(),
                      c->node_mem.as<long long>(), c->node_gpu.as<long long>()};
    bi.sched[0] = c->sched.as<long long>(); bi.sched[1] = c->sched.as<long long>() + N; bi.sched[2] = c->sched.as<long long>() + 2 * N;
    bi.n_nodes = N32;
    bi.seg_off = d_seg;
    bi.nodes = d_seg ? d_seg + G + 1 : nullptr;
    bi.n_part = n_part;
    gp_eff_base<<<(unsigned)((size_t)n_part * G), TH, 0, st>>>(bi, ar.ptr(part), d_err);
    gp_eff_finish<<<(unsigned)G, TH, 0, st>>>(ar.ptr(part), n_part, ar.ptr(base));
    ri.av = bi.av;
    for (int k = 0; k < 3; ++k) ri.sched[k] = bi.sched[k];
    ri.count = ar.ptr(cnt); ri.off = ar.ptr(off_p); ri.exec = ar.ptr(exe); ri.base = ar.ptr(base);
    ri.seg_off = d_seg;
    ri.n_apps = Q; ri.n_nodes = N32;
    ri.executors_reserved = algo == GP_MINIMAL_FRAGMENTATION ? 0 : 1;
    ri.charged = (int32_t)charged;
    gp_eff_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, ar.ptr(avg), d_err);
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    ar.get(avg_out, avg);
    ar.get(&herr, err);
    GP_TRY(ar.sync(c));
    return refuse(c, herr, kEffRefusals, who);
}

extern "C" {

gp_status gp_packing_efficiency(gp_ctx* c, const gp_apps* a, gp_algo algo, const gp_results* placed, gp_mode charged, double* avg_out) {
    if (!enter(c)) return GP_ERR_INVALID;
    return packing_efficiency(c, a, algo, placed, charged, nullptr, 1, avg_out, "gp_packing_efficiency");
}

// the same metric with row i averaged over its instance group's nodes (selectDriverNode's metadata) instead of the table's
gp_status gp_packing_efficiency_groups(gp_ctx* c, const gp_apps* a, gp_algo algo, const gp_results* placed, gp_mode charged,
                                       const int32_t* instance_group, int32_t n_instance_groups, double* avg_out) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!instance_group && c->n_nodes > 0) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency_groups: instance_group is NULL");
    static const int32_t none = -1;                     // an empty node table: no node in any instance group
    return packing_efficiency(c, a, algo, placed, charged, instance_group ? instance_group : &none, n_instance_groups, avg_out,
                              "gp_packing_efficiency_groups");
}
}  // extern "C"
