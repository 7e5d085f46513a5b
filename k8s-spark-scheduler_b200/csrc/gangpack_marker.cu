// gangpack_marker.cu -- the unschedulable-pod marker's capacity checks (gp_exceeds_cluster_capacity, with required node
// affinity gp_exceeds_cluster_capacity_affinity, their *_resident forms over the overhead table, and
// gp_exceeds_cluster_capacity_affinity_label_table over both it and the label table, the node-table forms, and
// gp_exceeds_cluster_capacity_driver_table over the driver table's stale rows), gp_match_node_affinity[_resident], and the
// overhead computer (gp_node_overhead).
#include "gangpack_ctx.cuh"
#include "gangpack_affinity.cuh"
#include "gangpack_capacity.cuh"
#include "gangpack_overhead.cuh"

#include <algorithm>
#include <string>
#include <vector>

// ---- required node affinity and the marker's capacity checks (gangpack_affinity.cuh, gangpack_capacity.cuh) ---------------
static bool csr_ok(const int64_t* off, int64_t n) {     // off[0] = 0, non-decreasing
    if (off[0] != 0) return false;
    for (int64_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
    return true;
}

// Host checks of the affinity programs (small) against n nodes and the label id ranges n_keys / n_values
static gp_status check_programs(gp_ctx* c, int32_t n, int32_t n_keys, int32_t n_values, const gp_node_affinities* P, const char* who) {
    auto bad = [&](const char* what) { return fail(c, GP_ERR_INVALID, who, what); };
    if (!P || P->n_aff < 0 || !P->sel_off || !P->term_off || !P->term_req_off || !P->req_val_off || (P->n_aff > 0 && !P->has_required))
        return bad("missing arrays or negative sizes");
    const int32_t A = P->n_aff;
    if (!csr_ok(P->sel_off, A) || !csr_ok(P->term_off, A)) return bad("sel_off or term_off does not start at 0 or decreases");
    const int64_t ns = P->sel_off[A], nt = P->term_off[A];
    if (!csr_ok(P->term_req_off, nt)) return bad("term_req_off does not start at 0 or decreases");
    const int64_t nr = P->term_req_off[nt];
    if (!csr_ok(P->req_val_off, nr)) return bad("req_val_off does not start at 0 or decreases");
    const int64_t nv = P->req_val_off[nr];
    if ((ns > 0 && (!P->sel_key || !P->sel_val)) || (nr > 0 && (!P->req_op || !P->req_key || !P->req_int)) || (nv > 0 && !P->req_val))
        return bad("missing arrays or negative sizes");
    for (int64_t t = 0; t < ns; ++t)
        if (P->sel_key[t] < 0 || P->sel_key[t] >= n_keys || P->sel_val[t] < 0 || P->sel_val[t] >= n_values)
            return bad("node selector key or value id out of range");
    for (int64_t r = 0; r < nr; ++r) {
        const int32_t op = P->req_op[r];
        if (op < GP_AFF_IN || op > GP_AFF_FIELD_NAME_NOT_IN) return bad("requirement operator out of range");
        if (op >= GP_AFF_FIELD_NAME_IN) {
            if (P->req_int[r] < -1 || P->req_int[r] >= n) return bad("metadata.name node index out of range (-1 or 0..n_nodes-1)");
            continue;
        }
        if (P->req_key[r] < 0 || P->req_key[r] >= n_keys) return bad("requirement key id out of range");
        for (int64_t v = P->req_val_off[r]; v < P->req_val_off[r + 1]; ++v) {
            if (P->req_val[v] < 0 || P->req_val[v] >= n_values) return bad("requirement value id out of range");
            if (v > P->req_val_off[r] && P->req_val[v] <= P->req_val[v - 1]) return bad("requirement values not strictly ascending");
        }
    }
    return GP_OK;
}

// Host checks of the per-call label offsets, then of the programs against them; each label entry is checked by
// gp_aff_labels on the device
static gp_status check_affinity(gp_ctx* c, const gp_node_labels* L, const gp_node_affinities* P, const char* who) {
    if (!L || L->n_nodes < 0 || L->n_keys < 0 || L->n_values < 0 || !L->label_off || (L->label_int_ok && !L->label_int))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    const int32_t n = L->n_nodes;
    if (!csr_ok(L->label_off, n)) return fail(c, GP_ERR_INVALID, who, "label_off does not start at 0 or decreases");
    if (L->label_off[n] > 0 && (!L->label_key || !L->label_val)) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    return check_programs(c, n, L->n_keys, L->n_values, P, who);
}

// The same for a resident call: a live label table, the node ids present, the programs against the table's id ranges (each
// node id is checked by gp_aff_ids on the device)
static gp_status check_affinity(gp_ctx* c, const gp_resident_labels* L, const gp_node_affinities* P, const char* who) {
    if (!L || L->n_nodes < 0 || (L->n_nodes > 0 && !L->node_id)) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    GP_TRY(require(c, c->lt.need(), who));
    return check_programs(c, L->n_nodes, c->lt.size.n_keys, c->lt.size.n_values, P, who);
}

// The label check's status word (kAffErr* bits)
static const Refusal kAffRefusals[] = {
    {kAffErrLabelKey, GP_ERR_INVALID, "label key id out of range or the keys of a node not strictly ascending"},
    {kAffErrLabelVal, GP_ERR_INVALID, "label value id out of range"},
    {kAffErrNodeId, GP_ERR_INVALID, "a label-table node id outside [-1, n_node_ids)"},
};

// Device staging of the labels (per-call CSR, or the resident node ids: rl != NULL) and programs, and the match launches
struct AffStage {
    Piece<long long> loff, lint, soff, toff, troff, rint, rvoff;
    Piece<int32_t> lkey, lval, skey, sval, rop, rkey, rval, nm, ne, rid;
    Piece<uint8_t> lok, hreq, terr;
    Piece<int> err;
    int32_t n, A, words;
    bool resident = false;
    AffLabelsIn L{};
    AffLabelsResident R{};
    AffProgIn P{};

    void take(Arena& ar, const gp_node_labels* l, const gp_resident_labels* rl, const gp_node_affinities* p) {
        resident = rl != nullptr;
        n = resident ? rl->n_nodes : l->n_nodes; A = p->n_aff; words = (n + 31) / 32;
        const size_t nl = resident ? 0 : l->label_off[n], ns = p->sel_off[A], nt = p->term_off[A], nr = p->term_req_off[nt],
                     nv = p->req_val_off[nr];
        const size_t N1 = resident ? 0 : (size_t)n + 1, A1 = (size_t)A + 1;
        loff = ar.take<long long>(N1); lkey = ar.take<int32_t>(nl); lval = ar.take<int32_t>(nl); lok = ar.take<uint8_t>(nl);
        lint = ar.take<long long>(nl); rid = ar.take<int32_t>(resident ? (size_t)n : 0);
        soff = ar.take<long long>(A1); skey = ar.take<int32_t>(ns); sval = ar.take<int32_t>(ns); hreq = ar.take<uint8_t>(A);
        toff = ar.take<long long>(A1); troff = ar.take<long long>(nt + 1); terr = ar.take<uint8_t>(nt);
        rop = ar.take<int32_t>(nr); rkey = ar.take<int32_t>(nr); rint = ar.take<long long>(nr); rvoff = ar.take<long long>(nr + 1);
        rval = ar.take<int32_t>(nv);
        nm = ar.take<int32_t>(A); ne = ar.take<int32_t>(A); err = ar.take<int>(2);
    }
    // uploads (an absent column is zeroed), zeroes the counters and the error word, and checks the labels (or the resident
    // node ids) once, whatever the number of affinities
    gp_status upload(gp_ctx* c, Arena& ar, const gp_node_labels* l, const gp_resident_labels* rl, const gp_node_affinities* p) {
        if (resident) {
            const LtCols t = lt_cols(c);
            R.n = n; R.n_rows = c->lt.size.n_node_ids; R.stride = c->lt.size.max_labels;
            R.count = t.count; R.key = t.key; R.val = t.val; R.val_int_ok = t.vok; R.val_int = t.vint;
            R.node_id = ar.put(rid, rl->node_id);
        } else {
            L.n = n; L.n_keys = l->n_keys; L.n_values = l->n_values;
            L.off = ar.put_or_zero(loff, l->label_off); L.key = ar.put_or_zero(lkey, l->label_key); L.val = ar.put_or_zero(lval, l->label_val);
            const uint8_t* int_ok = ar.put_or_zero(lok, l->label_int_ok);
            L.int_ok = l->label_int_ok ? int_ok : nullptr;
            L.ival = ar.put_or_zero(lint, l->label_int);
        }
        P.n_aff = A;
        P.sel_off = ar.put_or_zero(soff, p->sel_off); P.sel_key = ar.put_or_zero(skey, p->sel_key); P.sel_val = ar.put_or_zero(sval, p->sel_val);
        P.has_required = ar.put_or_zero(hreq, p->has_required); P.term_off = ar.put_or_zero(toff, p->term_off);
        P.term_req_off = ar.put_or_zero(troff, p->term_req_off); P.term_err = ar.put_or_zero(terr, p->term_parse_error);
        P.req_op = ar.put_or_zero(rop, p->req_op); P.req_key = ar.put_or_zero(rkey, p->req_key); P.req_int = ar.put_or_zero(rint, p->req_int);
        P.req_val_off = ar.put_or_zero(rvoff, p->req_val_off); P.req_val = ar.put_or_zero(rval, p->req_val);
        ar.zero(nm);
        ar.zero(ne);
        ar.zero(err);
        GP_TRY(ar.check(c));
        const unsigned blocks = (unsigned)((n + kAffThreads - 1) / kAffThreads);
        if (n > 0 && resident) gp_aff_ids<<<blocks, kAffThreads, 0, ar.st>>>(R, ar.ptr(err));
        else if (n > 0) gp_aff_labels<<<blocks, kAffThreads, 0, ar.st>>>(L, ar.ptr(err));
        return GP_OK;
    }
    // affinities [a0, a0 + k) into member rows 0..k-1
    void match(const Arena& ar, uint32_t* member, int32_t a0, int32_t k) const {
        if (n == 0) return;
        AffOut out{member, ar.ptr(nm), ar.ptr(ne), words, a0};
        for (int32_t y = 0; y < k; y += 65535) {
            const dim3 grid((unsigned)((n + kAffThreads - 1) / kAffThreads), (unsigned)std::min(k - y, 65535));
            if (resident) gp_aff_match<<<grid, kAffThreads, 0, ar.st>>>(R, P, out, a0 + y);
            else gp_aff_match<<<grid, kAffThreads, 0, ar.st>>>(L, P, out, a0 + y);
        }
    }
};

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer; the node sets are the node_group classes (aff ==
// NULL) or the affinities' matches.  The overhead is nodes->overhead_* (resident false) or, resident, GetNonSchedulableOverhead
// of the overhead table's records on node id over_ids[i] (-1: none), summed into this call's scratch by the query's kernels.
// The affinities' labels are the per-call labels, or with rlabels the label table's rows.
// gather_err (the *_node_table entries): nodes' allocatable and zone_id are device columns gathered from the node and label
// tables, kept in range by the gather, whose status word is read in the one synchronise before the entry's own refusals.
// apps_on_device (the driver-table entry): a's six quantities, exe_count and group are device columns (DtStale), used in place;
// the groups are copied back with the results for affinity_error.
// capacity_check: the host checks alone (capacity_run's first step), for an entry that has device work to do between them and
// the run.
static gp_status capacity_check(gp_ctx* c, const char* who, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                                const gp_node_affinities* aff, const gp_apps* a, gp_binpacker packer, bool resident,
                                const int32_t* over_ids, const gp_resident_labels* rlabels, const uint8_t* exceeds) {
    if (!aff) {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || nodes->n_groups < 1 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !exceeds)))
            return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes (n_groups >= 1; n_zones >= 1 with zone_id)");
    } else {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count ||
                               !a->group || !exceeds)))
            return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes (group required; n_zones >= 1 with zone_id)");
        if (nodes->node_group) return fail(c, GP_ERR_INVALID, who, "node_group must be NULL: the node sets are the affinities' matches");
        if (rlabels ? rlabels->n_nodes != nodes->n_nodes : (!labels || labels->n_nodes != nodes->n_nodes))
            return fail(c, GP_ERR_INVALID, who, "labels->n_nodes != nodes->n_nodes");
        const gp_status s = rlabels ? check_affinity(c, rlabels, aff, who) : check_affinity(c, labels, aff, who);
        if (s != GP_OK) return s;
    }
    if ((int)packer < GP_BP_TIGHTLY_PACK || (int)packer > GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION) return fail(c, GP_ERR_INVALID, who, "unknown packer");
    const int32_t n = nodes->n_nodes;
    const int32_t Z = nodes->zone_id ? nodes->n_zones : 1, G = aff ? aff->n_aff : nodes->n_groups;
    if (!aff && (int64_t)(G + 1) * Z > (int64_t)INT32_MAX / 2) return fail(c, GP_ERR_INVALID, who, "(n_groups + 1) * n_zones too large");
    if (aff && (int64_t)Z > (int64_t)INT32_MAX / 2) return fail(c, GP_ERR_INVALID, who, "n_zones too large");
    if (resident && n > 0 && !over_ids) return fail(c, GP_ERR_INVALID, who, "overhead_node_id missing");
    if (resident) GP_TRY(require(c, c->oht.need(), who));
    return GP_OK;
}

static gp_status capacity_run(gp_ctx* c, const char* who, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                              const gp_node_affinities* aff, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds,
                              uint8_t* affinity_error, bool resident = false, const int32_t* over_ids = nullptr,
                              const gp_resident_labels* rlabels = nullptr, const int* gather_err = nullptr, bool apps_on_device = false) {
    GP_TRY(capacity_check(c, who, nodes, labels, aff, a, packer, resident, over_ids, rlabels, exceeds));
    const int32_t n = nodes->n_nodes, Q = a->n_apps;
    const int32_t Z = nodes->zone_id ? nodes->n_zones : 1, G = aff ? aff->n_aff : nodes->n_groups;
    // classes per chunk: node_group -> its own class and the all-nodes class; affinities -> as many as keep K n and K Z
    // within kCapEntries (at least one)
    const int32_t K = !aff ? 2 : (int32_t)std::max<int64_t>(1, std::min<int64_t>(std::max(G, 1), kCapEntries / std::max<int64_t>({(int64_t)n, (int64_t)Z, 1})));
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t N = (size_t)n, q = (size_t)Q, E = (size_t)K * N, B = aff ? (size_t)K * (size_t)Z : (size_t)(G + 1) * (size_t)Z;
    size_t H = 64;
    while (H < 2 * q) H <<= 1;                          // more slots than drivers: every probe ends
    const size_t n_segs = E / kCapSeg + B + 1;
    // buckets of more than kCapSeg nodes in a chunk: at most E / (kCapSeg + 1), whatever the number of zones
    const int32_t ms_stride = (int32_t)std::max<size_t>(1, E / ((size_t)kCapSeg + 1));
    const int32_t pairs_per_chunk = (int32_t)std::max<int64_t>(1, std::min<int64_t>(std::max(Q, 1), kCapSlotEntries / ms_stride));
    const size_t A = (size_t)pairs_per_chunk * (size_t)ms_stride;
    const size_t q1 = std::max<size_t>(q, 1);
    Arena ar{c->callbuf, st};
    // resident overhead: the query's six columns, GetNonSchedulableOverhead last
    const auto alloc = ar.take<long long>(3 * N), over = ar.take<long long>((resident ? 6 : 3) * N);
    const auto zone = ar.take<int32_t>(N), grp = ar.take<int32_t>(N), key = ar.take<int32_t>(E), rank = ar.take<int32_t>(E),
               zst = ar.take<int32_t>(N);
    const auto staged = ar.take<long long>(3 * N), sched = ar.take<long long>(3 * E);
    const auto bcnt = ar.take<int32_t>(B), boff = ar.take<int32_t>(B + 1), soff = ar.take<int32_t>(B + 1), moff = ar.take<int32_t>(B + 1);
    const auto segs = ar.take<CapSeg>(n_segs);
    const size_t qh = apps_on_device ? 0 : q;           // host columns staged
    const auto qp = ar.take<long long>(6 * qh);
    const auto cnt = ar.take<int32_t>(qh), ag = ar.take<int32_t>(qh);
    const auto hash = ar.take<CapEntry>(H);
    const auto pairs = ar.take<CapPair>(q);
    const auto n_pairs = ar.take<int32_t>(2);
    const auto err = ar.take<int>(2);
    const auto app_pair = ar.take<int32_t>(q);
    const auto pref = ar.take<long long>(q + 1);
    const auto slots = ar.take<CapSlot>(A);
    const auto tot = ar.take<unsigned long long>(q1);
    const auto most = ar.take<long long>(q1), zb = ar.take<long long>(q1);
    const auto d_out = ar.take<uint8_t>(q1);
    AffStage as{};
    Piece<uint32_t> member{0, 0};
    if (aff) { as.take(ar, labels, rlabels, aff); member = ar.take<uint32_t>((size_t)K * (size_t)as.words); }
    const size_t NR = resident ? N : 0;
    const auto oids = ar.take<int32_t>(NR), odir = ar.take<int32_t>(resident ? (size_t)c->oht.size.n_node_ids : 0);
    const auto oacc = ar.take<unsigned long long>(12 * NR), owarned = ar.take<unsigned long long>(resident ? 1 : 0);
    const auto oerr = ar.take<int>(resident ? 2 : 0);   // the directory's word, then the overhead query's
    ar.reserve();
    ar.zero(hash);
    ar.fill(n_pairs, err, 0);                           // adjacent: one memset clears both
    if (resident) {
        ar.fill(odir, 0xff);
        ar.fill(oacc, oerr, 0);
    }
    if (aff) GP_TRY(as.upload(c, ar, labels, rlabels, aff));
    CapScratch s{};
    s.key = ar.ptr(key); s.rank = ar.ptr(rank); s.zone = ar.ptr(zst); s.bucket_cnt = ar.ptr(bcnt);
    s.bucket_off = ar.ptr(boff); s.seg_off = ar.ptr(soff); s.ms_off = ar.ptr(moff);
    for (int d = 0; d < 3; ++d) { s.staged[d] = ar.ptr(staged) + d * N; s.sched[d] = ar.ptr(sched) + d * E; }
    s.segs = ar.ptr(segs); s.err = ar.ptr(err);
    s.Z = Z; s.G = G; s.n = n;
    const int T = 256;
    CapClassesIn ci{};
    if (n > 0) {
        CapNodesIn ni{};
        ni.n = n;
        const int64_t* cols[2][3] = {{nodes->alloc_cpu_milli, nodes->alloc_mem_bytes, nodes->alloc_gpu},
                                     {nodes->overhead_cpu_milli, nodes->overhead_mem_bytes, nodes->overhead_gpu}};
        for (int d = 0; d < 3; ++d) ni.alloc[d] = gather_err ? (const long long*)cols[0][d] : ar.put(alloc.part(d * N, N), cols[0][d]);
        if (!resident)
            for (int d = 0; d < 3; ++d) ni.over[d] = ar.put(over.part(d * N, N), cols[1][d]);
        const int32_t* d_oids = ar.put(oids, resident ? over_ids : nullptr);
        ni.zone = gather_err ? nodes->zone_id : ar.put(zone, nodes->zone_id);
        ni.group = ar.put(grp, nodes->node_group);
        ci.group = ni.group;
        GP_TRY(ar.check(c));
        if (resident) {
            int* e = ar.ptr(oerr);
            enqueue_resident_dir(st, n, d_oids, c->oht.size.n_node_ids, ar.ptr(odir), e);
            oht_enqueue_sums(c, st, ar.ptr(odir), n, ar.ptr(oacc), ar.ptr(owarned), ar.ptr(over), nullptr, e + 1);
            for (int d = 0; d < 3; ++d) ni.over[d] = ar.ptr(over.part((3 + d) * N, N));
        }
        gp_cc_nodes<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(ni, s);
    }
    CapAppsIn ai{};
    ai.n = Q;
    const int64_t* qcols[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    if (apps_on_device) {
        for (int t = 0; t < 6; ++t) ai.q[t] = (const long long*)qcols[t];
        ai.count = a->exe_count;
        ai.group = a->group;
    } else {
        for (int t = 0; t < 6; ++t) ai.q[t] = ar.put(qp.part(q * t, q), qcols[t]);
        ar.put(cnt, a->exe_count);
        ai.count = ar.ptr(cnt);
        if (Q > 0) ai.group = ar.put(ag, a->group);
    }
    ai.n_groups = G;
    ai.min_group = aff ? 0 : -1;
    ai.hash_mask = (uint32_t)(H - 1);
    GP_TRY(ar.check(c));
    if (Q > 0) gp_cc_intern<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(ai, ar.ptr(hash), ar.ptr(pairs), ar.ptr(n_pairs), ar.ptr(app_pair), s.err);
    CapPairOut po{ar.ptr(tot), ar.ptr(most), ar.ptr(zb)};
    CapPassIn pi{};
    pi.pairs = ar.ptr(pairs); pi.n_pairs = ar.ptr(n_pairs); pi.pref = ar.ptr(pref); pi.out = po;
    pi.slots = ar.ptr(slots); pi.ms_stride = ms_stride;
    const int pass_blocks = c->sm_count * 8;
    if (aff) { ci.member = ar.ptr(member); ci.words = as.words; }
    // node_group: one chunk of both entries of every node (a0 = -1); affinities: chunks of K classes, the last one possibly
    // shorter (none when there are no affinities: the nodes and drivers are still validated)
    const int32_t n_chunks = aff ? (G + K - 1) / K : 1;
    for (int32_t ch = 0; ch < n_chunks; ++ch) {
        const int32_t a0 = aff ? ch * K : -1, k = aff ? std::min(K, G - a0) : 2;
        s.a0 = a0; s.K = k; s.B = aff ? k * Z : (int32_t)B;
        if (aff) as.match(ar, ar.ptr(member), a0, k);
        ar.zero(bcnt.part(0, s.B));
        GP_TRY(ar.check(c));
        const size_t e = (size_t)k * N;
        if (n > 0) gp_cc_keys<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(ci, s);
        gp_cc_bucket_scan<<<1, 1024, 0, st>>>(s);
        if (n > 0) gp_cc_scatter<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(s);
        gp_cc_pair_scan<<<1, 1024, 0, st>>>(s, ar.ptr(pairs), ar.ptr(n_pairs), ar.ptr(pref), po);
        pi.s = s;
        // The number of pairs is only known on the device; chunks beyond it return at once.  One chunk unless the pairs
        // times the multi-segment buckets exceed kCapSlotEntries (100 000 pairs over 50 000 nodes: 2.4 million slots, two).
        for (int32_t p0 = 0; p0 < Q; p0 += pairs_per_chunk) {
            pi.p0 = p0; pi.p1 = (int32_t)std::min<int64_t>((int64_t)p0 + pairs_per_chunk, Q);
            if (e > (size_t)kCapSeg) gp_cc_clear<<<(unsigned)std::min<size_t>((A + T - 1) / T, (size_t)c->sm_count * 16), T, 0, st>>>(pi);
            gp_cc_pass<<<pass_blocks, kCapThreads, 0, st>>>(pi);
        }
    }
    if (Q > 0) gp_cc_decide<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(Q, ai.count, ar.ptr(app_pair), ar.ptr(pairs), po, (int32_t)packer, ar.ptr(d_out));
    GP_CUDA(c, cudaGetLastError());
    int herr = 0, aerr = 0, oerr_h[2] = {0, 0}, gather = 0;
    std::vector<int32_t> n_error(aff ? (size_t)G : 0);
    std::vector<int32_t> dev_group(apps_on_device && aff && affinity_error ? q : 0);
    ar.get(dev_group.data(), a->group, dev_group.size());
    ar.get(exceeds, ar.ptr(d_out), q);
    ar.get(&herr, s.err, 1);
    if (aff) {
        ar.get(&aerr, ar.ptr(as.err), 1);
        ar.get(n_error.data(), as.ne);
    }
    ar.get(oerr_h, oerr);
    if (gather_err) ar.get(&gather, gather_err, 1);
    GP_TRY(ar.sync(c));
    GP_TRY(nt_refusal(c, gather, who));
    if (oerr_h[0]) return fail(c, GP_ERR_INVALID, who, "an overhead_node_id out of range or given twice");
    GP_TRY(oht_sum_refusal(c, oerr_h[1], who));
    if (aff) GP_TRY(refuse(c, aerr, kAffRefusals, who));
    const Refusal cc_refusals[] = {                     // the capacity kernels' status word (kCcErr* bits)
        {kCcErrNegative, GP_ERR_INVALID, "negative resource request or exe_count"},
        {kCcErrGroup, GP_ERR_INVALID, aff ? "driver group out of range (0..n_aff-1)" : "driver group out of range (-1 or 0..n_groups-1)"},
        {kCcErrZone, GP_ERR_INVALID, "zone_id out of range"},
        {kCcErrNodeGroup, GP_ERR_INVALID, "node_group out of range (-1 or 0..n_groups-1)"},
        {kCcErrUnrepresentable, GP_ERR_UNREPRESENTABLE, "request >= 2^61"},
        {kCcErrNodeQuantity, GP_ERR_UNREPRESENTABLE, "|allocatable| or |overhead| >= 2^61"}};
    GP_TRY(refuse(c, herr, cc_refusals, who));
    if (aff && affinity_error) {
        const int32_t* group = apps_on_device ? dev_group.data() : a->group;
        for (int32_t i = 0; i < Q; ++i) affinity_error[i] = n_error[group[i]] > 0 ? 1 : 0;
    }
    return GP_OK;
}

extern "C" {

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer (EXT/unschedulablepods.go:132-166); see
// gangpack_capacity.cuh and DESIGN §2.2
gp_status gp_exceeds_cluster_capacity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds) {
    if (!enter(c)) return GP_ERR_INVALID;
    return capacity_run(c, "gp_exceeds_cluster_capacity", nodes, nullptr, nullptr, a, packer, exceeds, nullptr);
}

// the same over the nodes each driver's required affinity matches (gangpack_affinity.cuh), overlapping sets allowed
gp_status gp_exceeds_cluster_capacity_affinity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                                               const gp_node_affinities* affinities, const gp_apps* a, gp_binpacker packer,
                                               uint8_t* exceeds, uint8_t* affinity_error) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_exceeds_cluster_capacity_affinity";
    if (!affinities) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    return capacity_run(c, who, nodes, labels, affinities, a, packer, exceeds, affinity_error);
}

// the two with GetNonSchedulableOverhead from the context's resident overhead table, on the device (nodes->overhead_* ignored)
gp_status gp_exceeds_cluster_capacity_resident(gp_ctx* c, const gp_capacity_nodes* nodes, const int32_t* overhead_node_id, const gp_apps* a,
                                               gp_binpacker packer, uint8_t* exceeds) {
    if (!enter(c)) return GP_ERR_INVALID;
    return capacity_run(c, "gp_exceeds_cluster_capacity_resident", nodes, nullptr, nullptr, a, packer, exceeds, nullptr, true, overhead_node_id);
}

gp_status gp_exceeds_cluster_capacity_affinity_resident(gp_ctx* c, const gp_capacity_nodes* nodes, const int32_t* overhead_node_id,
                                                        const gp_node_labels* labels, const gp_node_affinities* affinities, const gp_apps* a,
                                                        gp_binpacker packer, uint8_t* exceeds, uint8_t* affinity_error) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_exceeds_cluster_capacity_affinity_resident";
    if (!affinities) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    return capacity_run(c, who, nodes, labels, affinities, a, packer, exceeds, affinity_error, true, overhead_node_id);
}

// the same with the labels read in place from the label table
gp_status gp_exceeds_cluster_capacity_affinity_label_table(gp_ctx* c, const gp_capacity_nodes* nodes, const int32_t* overhead_node_id,
                                                           const gp_resident_labels* labels, const gp_node_affinities* affinities,
                                                           const gp_apps* a, gp_binpacker packer, uint8_t* exceeds, uint8_t* affinity_error) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_exceeds_cluster_capacity_affinity_label_table";
    if (!affinities || !labels) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    return capacity_run(c, who, nodes, nullptr, affinities, a, packer, exceeds, affinity_error, true, overhead_node_id, labels);
}

// the node-table forms: nt_gather fills allocatable and zone_id on the device, then the resident / label-table path runs
static gp_capacity_nodes gathered_nodes(const gp_node_table_nodes* nodes, const NtGathered& g, const int32_t* node_group, int32_t n_groups) {
    gp_capacity_nodes cn{};
    cn.n_nodes = g.usage.n_nodes;
    cn.alloc_cpu_milli = g.usage.alloc_cpu_milli;
    cn.alloc_mem_bytes = g.usage.alloc_mem_bytes;
    cn.alloc_gpu = g.usage.alloc_gpu;
    cn.n_zones = nodes->n_zones;
    cn.zone_id = g.sort.zone_id;
    cn.n_groups = n_groups;
    cn.node_group = node_group;
    return cn;
}

gp_status gp_exceeds_cluster_capacity_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, const int32_t* node_group, int32_t n_groups,
                                                 const gp_apps* a, gp_binpacker packer, uint8_t* exceeds) {
    static const char* who = "gp_exceeds_cluster_capacity_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, nullptr, 1, false, who, &g, nullptr, false));
    const gp_capacity_nodes cn = gathered_nodes(nodes, g, node_group, n_groups);
    GP_TRY(capacity_run(c, who, &cn, nullptr, nullptr, a, packer, exceeds, nullptr, true, nodes->overhead_node_id, nullptr, g.err));
    return nt_outputs(c, nodes, g);
}

gp_status gp_exceeds_cluster_capacity_affinity_node_table(gp_ctx* c, const gp_node_table_nodes* nodes, const gp_node_affinities* affinities,
                                                          const gp_apps* a, gp_binpacker packer, uint8_t* exceeds, uint8_t* affinity_error) {
    static const char* who = "gp_exceeds_cluster_capacity_affinity_node_table";
    if (!enter(c)) return GP_ERR_INVALID;
    if (!affinities) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, nullptr, 1, false, who, &g, nullptr, false));
    const gp_capacity_nodes cn = gathered_nodes(nodes, g, nullptr, 0);
    const gp_resident_labels rl{nodes->n_nodes, 0, nodes->node_table_id};
    GP_TRY(capacity_run(c, who, &cn, nullptr, affinities, a, packer, exceeds, affinity_error, true, nodes->overhead_node_id, &rl, g.err));
    return nt_outputs(c, nodes, g);
}

// The marker's whole sweep from the driver table (DESIGN §2.14): the host checks of the affinity node-table entry and the
// sweep's own, the gather enqueued, the stale stage (one synchronise, its refusals), then the capacity run on the stale
// columns in place over the caller's programs plus one that matches every node (the drivers without an affinity).
gp_status gp_exceeds_cluster_capacity_driver_table(gp_ctx* c, const gp_node_table_nodes* nodes, const gp_node_affinities* affinities,
                                                   const gp_stale_sweep* sw, gp_binpacker packer) {
    static const char* who = "gp_exceeds_cluster_capacity_driver_table";
    if (!enter(c)) return GP_ERR_INVALID;
    if (!affinities) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    NtGathered g{};
    GP_TRY(nt_gather(c, nodes, nullptr, 1, false, who, &g, nullptr, false));
    const gp_capacity_nodes cn = gathered_nodes(nodes, g, nullptr, 0);
    const gp_resident_labels rl{nodes->n_nodes, 0, nodes->node_table_id};
    // the caller's programs and, appended, one with no nodeSelector and no required affinity (it matches every node); arrays
    // the check would refuse are passed on as they are, so that it refuses them as the affinity node-table entry does
    const gp_node_affinities* P = affinities;
    gp_node_affinities ext = *P;
    std::vector<int64_t> sel_off, term_off;
    std::vector<uint8_t> has_required;
    if (P->n_aff >= 0 && P->sel_off && P->term_off && (P->n_aff == 0 || P->has_required) && P->n_aff < INT32_MAX) {
        const int32_t A = P->n_aff;
        sel_off.assign(P->sel_off, P->sel_off + A + 1);
        sel_off.push_back(sel_off[A]);
        term_off.assign(P->term_off, P->term_off + A + 1);
        term_off.push_back(term_off[A]);
        has_required.assign(A + 1, 0);
        if (A > 0) std::copy(P->has_required, P->has_required + A, has_required.begin());
        ext.n_aff = A + 1;
        ext.sel_off = sel_off.data(); ext.term_off = term_off.data(); ext.has_required = has_required.data();
    }
    const gp_apps none{};
    GP_TRY(capacity_check(c, who, &cn, nullptr, &ext, &none, packer, true, nodes->overhead_node_id, &rl, nullptr));
    if (!sw || !sw->stale_slot || !sw->exceeds || !sw->outcome || !sw->n_stale || sw->cap < 0)
        return fail(c, GP_ERR_INVALID, who, "NULL sweep or outputs, or a negative cap");
    GP_TRY(require(c, c->dt.need(), who));
    DtStale ds{};
    GP_TRY(dt_stale_stage(c, sw, P->n_aff, who, &ds));
    gp_apps a{};
    a.n_apps = ds.n;
    a.drv_cpu_milli = ds.q[0]; a.drv_mem_bytes = ds.q[1]; a.drv_gpu = ds.q[2];
    a.exe_cpu_milli = ds.q[3]; a.exe_mem_bytes = ds.q[4]; a.exe_gpu = ds.q[5];
    a.exe_count = ds.count; a.group = ds.group;
    std::vector<uint8_t> aff_err((size_t)ds.n);
    GP_TRY(capacity_run(c, who, &cn, nullptr, &ext, &a, packer, sw->exceeds, aff_err.data(), true, nodes->overhead_node_id, &rl, g.err,
                        true));
    for (int32_t i = 0; i < ds.n; ++i) {           // outcome holds 2 (outside the model) or 0 from the stale stage
        if (sw->outcome[i] == 2) sw->exceeds[i] = 0;
        else sw->outcome[i] = aff_err[i] ? 1 : 0;
    }
    return nt_outputs(c, nodes, g);
}

// GetRequiredNodeAffinity(...).Match for every (affinity, node) over the per-call labels or (rl) the label table's rows
static gp_status match_run(gp_ctx* c, const char* who, const gp_node_labels* labels, const gp_resident_labels* rl,
                           const gp_node_affinities* affinities, gp_affinity_match* out) {
    gp_status s = rl ? check_affinity(c, rl, affinities, who) : check_affinity(c, labels, affinities, who);
    if (s != GP_OK) return s;
    if (!out) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    Arena ar{c->callbuf, st};
    AffStage as{};
    as.take(ar, labels, rl, affinities);
    const auto member = ar.take<uint32_t>((size_t)as.A * (size_t)as.words);
    ar.reserve();
    GP_TRY(as.upload(c, ar, labels, rl, affinities));
    as.match(ar, ar.ptr(member), 0, as.A);
    GP_CUDA(c, cudaGetLastError());
    int aerr = 0;
    ar.get(out->member, member);
    ar.get(out->n_match, as.nm);
    ar.get(out->n_error, as.ne);
    ar.get(&aerr, ar.ptr(as.err), 1);
    GP_TRY(ar.sync(c));
    return refuse(c, aerr, kAffRefusals, who);
}

// see gangpack_affinity.cuh
gp_status gp_match_node_affinity(gp_ctx* c, const gp_node_labels* labels, const gp_node_affinities* affinities, gp_affinity_match* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    return match_run(c, "gp_match_node_affinity", labels, nullptr, affinities, out);
}

gp_status gp_match_node_affinity_resident(gp_ctx* c, const gp_resident_labels* labels, const gp_node_affinities* affinities,
                                          gp_affinity_match* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    return match_run(c, "gp_match_node_affinity_resident", nullptr, labels, affinities, out);
}

// The overhead kernels' status word (kOhErr* bits)
static const Refusal kOhRefusals[] = {
    {kOhErrRange, GP_ERR_INVALID, "an id out of its range (node, app key, app id, name or query node)"},
    {kOhErrAppPair, GP_ERR_INVALID, "app_key and app_id disagree on -1"},
    {kOhErrDuplicate, GP_ERR_INVALID, "a query node id, rr_app_key or soft_app_id given twice"},
    {kOhErrNegative, GP_ERR_INVALID, "negative request"},
    {kOhErrRequest, GP_ERR_UNREPRESENTABLE, "request >= 2^61"},
    {kOhErrSum, GP_ERR_UNREPRESENTABLE, "a per-node sum >= 2^61"},
};

// The overhead computer's per-call side (EXT/overhead.go:105-153) for a list of nodes; see gangpack_overhead.cuh
gp_status gp_node_overhead(gp_ctx* c, const gp_overhead_pods* p, const gp_overhead_reservations* r, int32_t n_nodes,
                           const int32_t* node_ids, gp_overhead_out* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_node_overhead";
    if (!p || !r || !out || p->n_pods < 0 || p->n_node_ids < 0 || p->n_app_keys < 0 || p->n_app_ids < 0 || p->n_names < 0 ||
        r->n_rr < 0 || r->n_soft < 0 || n_nodes < 0 || (n_nodes > 0 && !node_ids) ||
        (p->n_pods > 0 && (!p->node_id || !p->req_cpu_milli || !p->req_mem_bytes || !p->app_key || !p->app_id || !p->name_id)) ||
        (r->n_rr > 0 && (!r->rr_app_key || !r->rr_pod_off)) || (r->n_soft > 0 && (!r->soft_app_id || !r->soft_pod_off)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    if (p->n_pods > INT32_MAX) return fail(c, GP_ERR_INVALID, who, "n_pods must be below 2^31");
    // CSR offsets (one per reservation: host-sized); the entries themselves are checked on the device
    auto entries = [](const int64_t* off, int32_t n, int64_t* total) {
        if (n == 0) { *total = 0; return !off || off[0] == 0; }
        if (off[0] != 0) return false;
        for (int32_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
        *total = off[n];
        return true;
    };
    int64_t er = 0, es = 0;
    if (!entries(r->rr_pod_off, r->n_rr, &er) || !entries(r->soft_pod_off, r->n_soft, &es))
        return fail(c, GP_ERR_INVALID, who, "rr_pod_off or soft_pod_off does not start at 0 or decreases");
    if ((er > 0 && !r->rr_pod_name) || (es > 0 && !r->soft_pod_name)) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    if (er + es > ((int64_t)1 << 30)) return fail(c, GP_ERR_INVALID, who, "more than 2^30 reservation entries");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t P = (size_t)p->n_pods, N = (size_t)n_nodes, R = (size_t)r->n_rr, S = (size_t)r->n_soft;
    size_t H = 64;
    while (H < 2 * (size_t)(er + es)) H <<= 1;           // at most half full: every probe ends
    // the overhead kernels' counter and status word, read back in one copy
    struct OhWord { unsigned long long n_warned; int err, unused; };
    Arena ar{c->callbuf, st};
    const auto node = ar.take<int32_t>(P);
    const auto req = ar.take<long long>(3 * P);
    const auto listed = ar.take<uint8_t>(P);
    const auto ak = ar.take<int32_t>(P), ai = ar.take<int32_t>(P), name = ar.take<int32_t>(P);
    const auto exe = ar.take<uint8_t>(P), spark = ar.take<uint8_t>(P), has = ar.take<uint8_t>(P);
    const auto rkey = ar.take<int32_t>(R);
    const auto roff = ar.take<long long>(R + 1);
    const auto rname = ar.take<int32_t>((size_t)er), skey = ar.take<int32_t>(S);
    const auto soff = ar.take<long long>(S + 1);
    const auto sname = ar.take<int32_t>((size_t)es), qn = ar.take<int32_t>(N);
    const auto rok = ar.take<int32_t>((size_t)p->n_app_keys), soa = ar.take<int32_t>((size_t)p->n_app_ids),
               ron = ar.take<int32_t>((size_t)p->n_node_ids);
    const auto set = ar.take<unsigned long long>(H), acc = ar.take<unsigned long long>(12 * N);
    const auto word = ar.take<OhWord>(1);
    const auto d_out = ar.take<long long>(6 * N);
    ar.reserve();
    // the directories and the hash set start at -1 / empty; the sums, n_warned and the error word at 0
    ar.fill(rok, set, 0xff);
    ar.fill(acc, word, 0);
    OhPodsIn pi{};
    pi.node_id = ar.put(node, p->node_id);
    const int64_t* reqs[3] = {p->req_cpu_milli, p->req_mem_bytes, p->req_gpu};
    for (int d = 0; d < 3; ++d) pi.req[d] = ar.put(req.part(P * d, P), reqs[d]);
    pi.listed = ar.put(listed, p->listed);
    pi.app_key = ar.put(ak, p->app_key); pi.app_id = ar.put(ai, p->app_id); pi.name_id = ar.put(name, p->name_id);
    pi.is_executor = ar.put(exe, p->is_executor);
    pi.spark_scheduler = ar.put(spark, p->spark_scheduler);
    pi.has_reservation = ar.ptr(has);
    ar.put(rkey, r->rr_app_key);
    if (R) ar.put(roff, r->rr_pod_off);
    ar.put(rname, r->rr_pod_name);
    ar.put(skey, r->soft_app_id);
    if (S) ar.put(soff, r->soft_pod_off);
    ar.put(sname, r->soft_pod_name);
    ar.put(qn, node_ids);
    GP_TRY(ar.check(c));
    OhMaps M{ar.ptr(rok), ar.ptr(soa), ar.ptr(ron), ar.ptr(set), (uint32_t)(H - 1), r->n_rr};
    int* d_err = &ar.ptr(word)->err;
    const int T = 256, cap = c->sm_count * 8;
    const long long n_dir = (long long)R + (long long)S + (long long)N;
    if (n_dir > 0) {
        OhDirIn D{r->n_rr, r->n_soft, n_nodes, p->n_app_keys, p->n_app_ids, p->n_node_ids, ar.ptr(rkey), ar.ptr(skey), ar.ptr(qn)};
        gp_oh_dir<<<(unsigned)std::min<long long>((n_dir + T - 1) / T, cap), T, 0, st>>>(D, M, d_err);
    }
    if (er + es > 0) {
        OhSetIn si{ar.ptr(roff), ar.ptr(rname), ar.ptr(soff), ar.ptr(sname), r->n_rr, r->n_soft, p->n_names, (long long)er, (long long)es};
        gp_oh_insert<<<(unsigned)std::min<long long>((er + es + T - 1) / T, cap), T, 0, st>>>(si, M, d_err);
    }
    OhAcc A{ar.ptr(acc), &ar.ptr(word)->n_warned, n_nodes};
    if (P > 0) {
        pi.n = (long long)P; pi.n_node_ids = p->n_node_ids; pi.n_app_keys = p->n_app_keys; pi.n_app_ids = p->n_app_ids; pi.n_names = p->n_names;
        gp_oh_pods<<<(unsigned)((P + kOhThreads - 1) / kOhThreads), kOhThreads, 0, st>>>(pi, OhCallLookup{M}, A, d_err);
    }
    if (N > 0) gp_oh_finish<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(A, ar.ptr(d_out), d_err);
    GP_CUDA(c, cudaGetLastError());
    int64_t* outs[6] = {out->overhead_cpu_milli, out->overhead_mem_bytes, out->overhead_gpu,
                        out->nonsched_cpu_milli, out->nonsched_mem_bytes, out->nonsched_gpu};
    for (int k = 0; k < 6; ++k) ar.get(outs[k], d_out.part(N * k, N));
    ar.get(out->has_reservation, has);
    OhWord hw{};
    ar.get(&hw, word);
    GP_TRY(ar.sync(c));
    GP_TRY(refuse(c, hw.err, kOhRefusals, who));
    if (out->n_warned) *out->n_warned = (int64_t)hw.n_warned;
    return GP_OK;
}

}  // extern "C"
