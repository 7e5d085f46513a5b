// gangpack_marker.cu -- the unschedulable-pod marker's capacity checks (gp_exceeds_cluster_capacity, with required node
// affinity gp_exceeds_cluster_capacity_affinity), gp_match_node_affinity, and the overhead computer (gp_node_overhead).
#include "gangpack_ctx.cuh"
#include "gangpack_affinity.cuh"
#include "gangpack_capacity.cuh"
#include "gangpack_overhead.cuh"

#include <algorithm>
#include <string>
#include <vector>

// ---- required node affinity and the marker's capacity checks (gangpack_affinity.cuh, gangpack_capacity.cuh) ---------------
// Host checks of the label offsets and of the affinity programs (small); each label entry is checked by gp_aff_match itself.
static gp_status check_affinity(gp_ctx* c, const gp_node_labels* L, const gp_node_affinities* P, const char* who) {
    auto bad = [&](const char* what) { return fail(c, GP_ERR_INVALID, std::string(who) + ": " + what); };
    if (!L || !P || L->n_nodes < 0 || L->n_keys < 0 || L->n_values < 0 || P->n_aff < 0 || !L->label_off || !P->sel_off ||
        !P->term_off || !P->term_req_off || !P->req_val_off || (P->n_aff > 0 && !P->has_required) || (L->label_int_ok && !L->label_int))
        return bad("missing arrays or negative sizes");
    auto csr = [](const int64_t* off, int64_t n) {      // off[0] = 0, non-decreasing
        if (off[0] != 0) return false;
        for (int64_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
        return true;
    };
    const int32_t n = L->n_nodes, A = P->n_aff;
    if (!csr(L->label_off, n)) return bad("label_off does not start at 0 or decreases");
    if (L->label_off[n] > 0 && (!L->label_key || !L->label_val)) return bad("missing arrays or negative sizes");
    if (!csr(P->sel_off, A) || !csr(P->term_off, A)) return bad("sel_off or term_off does not start at 0 or decreases");
    const int64_t ns = P->sel_off[A], nt = P->term_off[A];
    if (!csr(P->term_req_off, nt)) return bad("term_req_off does not start at 0 or decreases");
    const int64_t nr = P->term_req_off[nt];
    if (!csr(P->req_val_off, nr)) return bad("req_val_off does not start at 0 or decreases");
    const int64_t nv = P->req_val_off[nr];
    if ((ns > 0 && (!P->sel_key || !P->sel_val)) || (nr > 0 && (!P->req_op || !P->req_key || !P->req_int)) || (nv > 0 && !P->req_val))
        return bad("missing arrays or negative sizes");
    for (int64_t t = 0; t < ns; ++t)
        if (P->sel_key[t] < 0 || P->sel_key[t] >= L->n_keys || P->sel_val[t] < 0 || P->sel_val[t] >= L->n_values)
            return bad("node selector key or value id out of range");
    for (int64_t r = 0; r < nr; ++r) {
        const int32_t op = P->req_op[r];
        if (op < GP_AFF_IN || op > GP_AFF_FIELD_NAME_NOT_IN) return bad("requirement operator out of range");
        if (op >= GP_AFF_FIELD_NAME_IN) {
            if (P->req_int[r] < -1 || P->req_int[r] >= n) return bad("metadata.name node index out of range (-1 or 0..n_nodes-1)");
            continue;
        }
        if (P->req_key[r] < 0 || P->req_key[r] >= L->n_keys) return bad("requirement key id out of range");
        for (int64_t v = P->req_val_off[r]; v < P->req_val_off[r + 1]; ++v) {
            if (P->req_val[v] < 0 || P->req_val[v] >= L->n_values) return bad("requirement value id out of range");
            if (v > P->req_val_off[r] && P->req_val[v] <= P->req_val[v - 1]) return bad("requirement values not strictly ascending");
        }
    }
    return GP_OK;
}

// Device staging of the labels and programs, and the match launches
struct AffStage {
    size_t o_loff, o_lkey, o_lval, o_lok, o_lint, o_soff, o_skey, o_sval, o_hreq, o_toff, o_troff, o_terr, o_rop, o_rkey, o_rint,
        o_rvoff, o_rval, o_nm, o_ne, o_err;
    int64_t nl, ns, nt, nr, nv;
    int32_t n, A, words;
    AffLabelsIn L{};
    AffProgIn P{};

    void take(Arena& ar, const gp_node_labels* l, const gp_node_affinities* p) {
        n = l->n_nodes; A = p->n_aff; words = (n + 31) / 32;
        nl = l->label_off[n]; ns = p->sel_off[A]; nt = p->term_off[A]; nr = p->term_req_off[nt]; nv = p->req_val_off[nr];
        const size_t N1 = (size_t)n + 1, A1 = (size_t)A + 1;
        o_loff = ar.take(8 * N1); o_lkey = ar.take(4 * nl); o_lval = ar.take(4 * nl); o_lok = ar.take(nl); o_lint = ar.take(8 * nl);
        o_soff = ar.take(8 * A1); o_skey = ar.take(4 * ns); o_sval = ar.take(4 * ns); o_hreq = ar.take(A);
        o_toff = ar.take(8 * A1); o_troff = ar.take(8 * (nt + 1)); o_terr = ar.take(nt);
        o_rop = ar.take(4 * nr); o_rkey = ar.take(4 * nr); o_rint = ar.take(8 * nr); o_rvoff = ar.take(8 * (nr + 1)); o_rval = ar.take(4 * nv);
        o_nm = ar.take(4 * (size_t)A); o_ne = ar.take(4 * (size_t)A); o_err = ar.take(8);
    }
    // uploads, zeroes the counters and the error word
    cudaError_t upload(const Arena& ar, const gp_node_labels* l, const gp_node_affinities* p, cudaStream_t st) {
        char* b = ar.base();
        struct Piece { size_t o; const void* src; size_t bytes; };
        const Piece pieces[] = {
            {o_loff, l->label_off, 8 * ((size_t)n + 1)}, {o_lkey, l->label_key, 4 * (size_t)nl}, {o_lval, l->label_val, 4 * (size_t)nl},
            {o_lok, l->label_int_ok, (size_t)nl}, {o_lint, l->label_int, 8 * (size_t)nl},
            {o_soff, p->sel_off, 8 * ((size_t)A + 1)}, {o_skey, p->sel_key, 4 * (size_t)ns}, {o_sval, p->sel_val, 4 * (size_t)ns},
            {o_hreq, p->has_required, (size_t)A}, {o_toff, p->term_off, 8 * ((size_t)A + 1)},
            {o_troff, p->term_req_off, 8 * ((size_t)nt + 1)}, {o_terr, p->term_parse_error, (size_t)nt},
            {o_rop, p->req_op, 4 * (size_t)nr}, {o_rkey, p->req_key, 4 * (size_t)nr}, {o_rint, p->req_int, 8 * (size_t)nr},
            {o_rvoff, p->req_val_off, 8 * ((size_t)nr + 1)}, {o_rval, p->req_val, 4 * (size_t)nv}};
        for (const Piece& pc : pieces) {
            if (pc.bytes == 0) continue;
            const cudaError_t e = pc.src ? ar.upload(pc.o, pc.src, pc.bytes, st) : cudaMemsetAsync(b + pc.o, 0, pc.bytes, st);
            if (e != cudaSuccess) return e;
        }
        L.n = n; L.n_keys = l->n_keys; L.n_values = l->n_values;
        L.off = (const long long*)(b + o_loff); L.key = (const int32_t*)(b + o_lkey); L.val = (const int32_t*)(b + o_lval);
        L.int_ok = l->label_int_ok ? (const uint8_t*)(b + o_lok) : nullptr; L.ival = (const long long*)(b + o_lint);
        P.n_aff = A;
        P.sel_off = (const long long*)(b + o_soff); P.sel_key = (const int32_t*)(b + o_skey); P.sel_val = (const int32_t*)(b + o_sval);
        P.has_required = (const uint8_t*)(b + o_hreq); P.term_off = (const long long*)(b + o_toff);
        P.term_req_off = (const long long*)(b + o_troff); P.term_err = (const uint8_t*)(b + o_terr);
        P.req_op = (const int32_t*)(b + o_rop); P.req_key = (const int32_t*)(b + o_rkey); P.req_int = (const long long*)(b + o_rint);
        P.req_val_off = (const long long*)(b + o_rvoff); P.req_val = (const int32_t*)(b + o_rval);
        // n_match, n_error and the error word; the labels are checked once here, whatever the number of affinities
        cudaError_t e = cudaMemsetAsync(b + o_nm, 0, 4 * (size_t)A, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b + o_ne, 0, 4 * (size_t)A, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b + o_err, 0, 8, st);
        if (e == cudaSuccess && n > 0) gp_aff_labels<<<(unsigned)((n + kAffThreads - 1) / kAffThreads), kAffThreads, 0, st>>>(L, (int*)(b + o_err));
        return e;
    }
    // affinities [a0, a0 + k) into member rows 0..k-1
    void match(const Arena& ar, uint32_t* member, int32_t a0, int32_t k, cudaStream_t st) const {
        if (n == 0) return;
        char* b = ar.base();
        AffOut out{member, (int32_t*)(b + o_nm), (int32_t*)(b + o_ne), words, a0};
        for (int32_t y = 0; y < k; y += 65535) {
            const dim3 grid((unsigned)((n + kAffThreads - 1) / kAffThreads), (unsigned)std::min(k - y, 65535));
            gp_aff_match<<<grid, kAffThreads, 0, st>>>(L, P, out, a0 + y);
        }
    }
    gp_status label_error(gp_ctx* c, int herr, const char* who) const {
        if (herr & kAffErrLabelKey) return fail(c, GP_ERR_INVALID, std::string(who) + ": label key id out of range or the keys of a node not strictly ascending");
        if (herr & kAffErrLabelVal) return fail(c, GP_ERR_INVALID, std::string(who) + ": label value id out of range");
        return GP_OK;
    }
};

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer; the node sets are the node_group classes (aff ==
// NULL) or the affinities' matches
static gp_status capacity_run(gp_ctx* c, const char* who, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                              const gp_node_affinities* aff, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds,
                              uint8_t* affinity_error) {
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    if (!aff) {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || nodes->n_groups < 1 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !exceeds)))
            return bad(GP_ERR_INVALID, "missing arrays or bad sizes (n_groups >= 1; n_zones >= 1 with zone_id)");
    } else {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count ||
                               !a->group || !exceeds)))
            return bad(GP_ERR_INVALID, "missing arrays or bad sizes (group required; n_zones >= 1 with zone_id)");
        if (nodes->node_group) return bad(GP_ERR_INVALID, "node_group must be NULL: the node sets are the affinities' matches");
        if (!labels || labels->n_nodes != nodes->n_nodes) return bad(GP_ERR_INVALID, "labels->n_nodes != nodes->n_nodes");
        const gp_status s = check_affinity(c, labels, aff, who);
        if (s != GP_OK) return s;
    }
    if ((int)packer < GP_BP_TIGHTLY_PACK || (int)packer > GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION) return bad(GP_ERR_INVALID, "unknown packer");
    const int32_t n = nodes->n_nodes, Q = a->n_apps;
    const int32_t Z = nodes->zone_id ? nodes->n_zones : 1, G = aff ? aff->n_aff : nodes->n_groups;
    if (!aff && (int64_t)(G + 1) * Z > (int64_t)INT32_MAX / 2) return bad(GP_ERR_INVALID, "(n_groups + 1) * n_zones too large");
    if (aff && (int64_t)Z > (int64_t)INT32_MAX / 2) return bad(GP_ERR_INVALID, "n_zones too large");
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
    Arena ar{c->capprep};
    const size_t o_alloc = ar.take(24 * N), o_over = ar.take(24 * N), o_zone = ar.take(4 * N), o_grp = ar.take(4 * N), o_key = ar.take(4 * E),
                 o_rank = ar.take(4 * E), o_zst = ar.take(4 * N), o_staged = ar.take(24 * N), o_sched = ar.take(24 * E), o_bcnt = ar.take(4 * B),
                 o_boff = ar.take(4 * (B + 1)), o_soff = ar.take(4 * (B + 1)), o_moff = ar.take(4 * (B + 1)), o_segs = ar.take(sizeof(CapSeg) * n_segs),
                 o_q = ar.take(48 * q), o_cnt = ar.take(4 * q), o_ag = ar.take(4 * q), o_hash = ar.take(sizeof(CapEntry) * H),
                 o_pairs = ar.take(sizeof(CapPair) * q), o_np = ar.take(8), o_err = ar.take(8), o_ap = ar.take(4 * q),
                 o_pref = ar.take(8 * (q + 1)), o_slots = ar.take(sizeof(CapSlot) * A), o_T = ar.take(8 * q1),
                 o_M = ar.take(8 * q1), o_zb = ar.take(8 * q1), o_out = ar.take(q1);
    AffStage as{};
    size_t o_member = 0;
    if (aff) { as.take(ar, labels, aff); o_member = ar.take(4 * (size_t)K * (size_t)as.words); }
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    // n_pairs and the error word are adjacent: one memset clears both
    GP_CUDA(c, cudaMemsetAsync(b + o_hash, 0, sizeof(CapEntry) * H, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_np, 0, o_ap - o_np, st));
    if (aff) GP_CUDA(c, as.upload(ar, labels, aff, st));
    CapScratch s{};
    s.key = (int32_t*)(b + o_key); s.rank = (int32_t*)(b + o_rank); s.zone = (int32_t*)(b + o_zst); s.bucket_cnt = (int32_t*)(b + o_bcnt);
    s.bucket_off = (int32_t*)(b + o_boff); s.seg_off = (int32_t*)(b + o_soff); s.ms_off = (int32_t*)(b + o_moff);
    for (int d = 0; d < 3; ++d) { s.staged[d] = (long long*)(b + o_staged) + d * N; s.sched[d] = (long long*)(b + o_sched) + d * E; }
    s.segs = (CapSeg*)(b + o_segs); s.err = (int*)(b + o_err);
    s.Z = Z; s.G = G; s.n = n;
    const int T = 256;
    CapClassesIn ci{};
    if (n > 0) {
        CapNodesIn ni{};
        ni.n = n;
        const int64_t* cols[6] = {nodes->alloc_cpu_milli, nodes->alloc_mem_bytes, nodes->alloc_gpu,
                                  nodes->overhead_cpu_milli, nodes->overhead_mem_bytes, nodes->overhead_gpu};
        for (int d = 0; d < 6; ++d) {
            if (!cols[d]) continue;
            const size_t o = (d < 3 ? o_alloc : o_over) + 8 * N * (size_t)(d % 3);
            GP_CUDA(c, ar.upload(o, cols[d], 8 * N, st));
            (d < 3 ? ni.alloc : ni.over)[d % 3] = (const long long*)(b + o);
        }
        if (nodes->zone_id) { GP_CUDA(c, ar.upload(o_zone, nodes->zone_id, 4 * N, st)); ni.zone = (const int32_t*)(b + o_zone); }
        if (nodes->node_group) { GP_CUDA(c, ar.upload(o_grp, nodes->node_group, 4 * N, st)); ni.group = (const int32_t*)(b + o_grp); }
        ci.group = ni.group;
        gp_cc_nodes<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(ni, s);
    }
    CapAppsIn ai{};
    ai.n = Q;
    const int64_t* qcols[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    for (int t = 0; t < 6; ++t) {
        if (!qcols[t]) continue;
        GP_CUDA(c, ar.upload(o_q + 8 * q * (size_t)t, qcols[t], 8 * q, st));
        ai.q[t] = (const long long*)(b + o_q) + q * (size_t)t;
    }
    if (Q > 0) GP_CUDA(c, ar.upload(o_cnt, a->exe_count, 4 * q, st));
    ai.count = (const int32_t*)(b + o_cnt);
    if (a->group && Q > 0) { GP_CUDA(c, ar.upload(o_ag, a->group, 4 * q, st)); ai.group = (const int32_t*)(b + o_ag); }
    ai.n_groups = G;
    ai.min_group = aff ? 0 : -1;
    ai.hash_mask = (uint32_t)(H - 1);
    CapPair* pairs = (CapPair*)(b + o_pairs);
    int32_t* n_pairs = (int32_t*)(b + o_np);
    int32_t* app_pair = (int32_t*)(b + o_ap);
    if (Q > 0) gp_cc_intern<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(ai, (CapEntry*)(b + o_hash), pairs, n_pairs, app_pair, s.err);
    long long* pref = (long long*)(b + o_pref);
    CapPairOut po{(unsigned long long*)(b + o_T), (long long*)(b + o_M), (long long*)(b + o_zb)};
    CapPassIn pi{};
    pi.pairs = pairs; pi.n_pairs = n_pairs; pi.pref = pref; pi.out = po;
    pi.slots = (CapSlot*)(b + o_slots); pi.ms_stride = ms_stride;
    const int pass_blocks = c->sm_count * 8;
    if (aff) { ci.member = (const uint32_t*)(b + o_member); ci.words = as.words; }
    // node_group: one chunk of both entries of every node (a0 = -1); affinities: chunks of K classes, the last one possibly
    // shorter (none when there are no affinities: the nodes and drivers are still validated)
    const int32_t n_chunks = aff ? (G + K - 1) / K : 1;
    for (int32_t ch = 0; ch < n_chunks; ++ch) {
        const int32_t a0 = aff ? ch * K : -1, k = aff ? std::min(K, G - a0) : 2;
        s.a0 = a0; s.K = k; s.B = aff ? k * Z : (int32_t)B;
        if (aff) as.match(ar, (uint32_t*)(b + o_member), a0, k, st);
        GP_CUDA(c, cudaMemsetAsync(s.bucket_cnt, 0, 4 * (size_t)s.B, st));
        const size_t e = (size_t)k * N;
        if (n > 0) gp_cc_keys<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(ci, s);
        gp_cc_bucket_scan<<<1, 1024, 0, st>>>(s);
        if (n > 0) gp_cc_scatter<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(s);
        gp_cc_pair_scan<<<1, 1024, 0, st>>>(s, pairs, n_pairs, pref, po);
        pi.s = s;
        // The number of pairs is only known on the device; chunks beyond it return at once.  One chunk unless the pairs
        // times the multi-segment buckets exceed kCapSlotEntries (100 000 pairs over 50 000 nodes: 2.4 million slots, two).
        for (int32_t p0 = 0; p0 < Q; p0 += pairs_per_chunk) {
            pi.p0 = p0; pi.p1 = (int32_t)std::min<int64_t>((int64_t)p0 + pairs_per_chunk, Q);
            if (e > (size_t)kCapSeg) gp_cc_clear<<<(unsigned)std::min<size_t>((A + T - 1) / T, (size_t)c->sm_count * 16), T, 0, st>>>(pi);
            gp_cc_pass<<<pass_blocks, kCapThreads, 0, st>>>(pi);
        }
    }
    uint8_t* d_out = (uint8_t*)(b + o_out);
    if (Q > 0) gp_cc_decide<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(Q, ai.count, app_pair, pairs, po, (int32_t)packer, d_out);
    GP_CUDA(c, cudaGetLastError());
    int herr = 0, aerr = 0;
    std::vector<int32_t> n_error(aff ? (size_t)G : 0);
    if (Q > 0) GP_CUDA(c, cudaMemcpyAsync(exceeds, d_out, q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&herr, s.err, 4, cudaMemcpyDeviceToHost, st));
    if (aff) {
        GP_CUDA(c, cudaMemcpyAsync(&aerr, b + as.o_err, 4, cudaMemcpyDeviceToHost, st));
        if (G > 0) GP_CUDA(c, cudaMemcpyAsync(n_error.data(), b + as.o_ne, 4 * (size_t)G, cudaMemcpyDeviceToHost, st));
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (aff) { const gp_status ls = as.label_error(c, aerr, who); if (ls != GP_OK) return ls; }
    if (herr & kCcErrNegative) return bad(GP_ERR_INVALID, "negative resource request or exe_count");
    if (herr & kCcErrGroup) return bad(GP_ERR_INVALID, aff ? "driver group out of range (0..n_aff-1)" : "driver group out of range (-1 or 0..n_groups-1)");
    if (herr & kCcErrZone) return bad(GP_ERR_INVALID, "zone_id out of range");
    if (herr & kCcErrNodeGroup) return bad(GP_ERR_INVALID, "node_group out of range (-1 or 0..n_groups-1)");
    if (herr & kCcErrUnrepresentable) return bad(GP_ERR_UNREPRESENTABLE, "request >= 2^61");
    if (herr & kCcErrNodeQuantity) return bad(GP_ERR_UNREPRESENTABLE, "|allocatable| or |overhead| >= 2^61");
    if (aff && affinity_error)
        for (int32_t i = 0; i < Q; ++i) affinity_error[i] = n_error[a->group[i]] > 0 ? 1 : 0;
    return GP_OK;
}

extern "C" {

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer (EXT/unschedulablepods.go:132-166); see
// gangpack_capacity.cuh and DESIGN §2.2
gp_status gp_exceeds_cluster_capacity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds) {
    if (!c) return GP_ERR_INVALID;
    return capacity_run(c, "gp_exceeds_cluster_capacity", nodes, nullptr, nullptr, a, packer, exceeds, nullptr);
}

// the same over the nodes each driver's required affinity matches (gangpack_affinity.cuh), overlapping sets allowed
gp_status gp_exceeds_cluster_capacity_affinity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                                               const gp_node_affinities* affinities, const gp_apps* a, gp_binpacker packer,
                                               uint8_t* exceeds, uint8_t* affinity_error) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_exceeds_cluster_capacity_affinity";
    if (!affinities) return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or negative sizes");
    return capacity_run(c, who, nodes, labels, affinities, a, packer, exceeds, affinity_error);
}

// GetRequiredNodeAffinity(...).Match for every (affinity, node); see gangpack_affinity.cuh
gp_status gp_match_node_affinity(gp_ctx* c, const gp_node_labels* labels, const gp_node_affinities* affinities, gp_affinity_match* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_match_node_affinity";
    gp_status s = check_affinity(c, labels, affinities, who);
    if (s != GP_OK) return s;
    if (!out) return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or negative sizes");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    Arena ar{c->capprep};
    AffStage as{};
    as.take(ar, labels, affinities);
    const size_t mbytes = 4 * (size_t)as.A * (size_t)as.words;
    const size_t o_member = ar.take(mbytes);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, as.upload(ar, labels, affinities, st));
    as.match(ar, (uint32_t*)(b + o_member), 0, as.A, st);
    GP_CUDA(c, cudaGetLastError());
    int aerr = 0;
    if (out->member && mbytes) GP_CUDA(c, cudaMemcpyAsync(out->member, b + o_member, mbytes, cudaMemcpyDeviceToHost, st));
    if (out->n_match && as.A) GP_CUDA(c, cudaMemcpyAsync(out->n_match, b + as.o_nm, 4 * (size_t)as.A, cudaMemcpyDeviceToHost, st));
    if (out->n_error && as.A) GP_CUDA(c, cudaMemcpyAsync(out->n_error, b + as.o_ne, 4 * (size_t)as.A, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&aerr, b + as.o_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return as.label_error(c, aerr, who);
}

// The overhead computer's per-call side (EXT/overhead.go:105-153) for a list of nodes; see gangpack_overhead.cuh
gp_status gp_node_overhead(gp_ctx* c, const gp_overhead_pods* p, const gp_overhead_reservations* r, int32_t n_nodes,
                           const int32_t* node_ids, gp_overhead_out* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_node_overhead";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    if (!p || !r || !out || p->n_pods < 0 || p->n_node_ids < 0 || p->n_app_keys < 0 || p->n_app_ids < 0 || p->n_names < 0 ||
        r->n_rr < 0 || r->n_soft < 0 || n_nodes < 0 || (n_nodes > 0 && !node_ids) ||
        (p->n_pods > 0 && (!p->node_id || !p->req_cpu_milli || !p->req_mem_bytes || !p->app_key || !p->app_id || !p->name_id)) ||
        (r->n_rr > 0 && (!r->rr_app_key || !r->rr_pod_off)) || (r->n_soft > 0 && (!r->soft_app_id || !r->soft_pod_off)))
        return bad(GP_ERR_INVALID, "missing arrays or negative sizes");
    if (p->n_pods > INT32_MAX) return bad(GP_ERR_INVALID, "n_pods must be below 2^31");
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
        return bad(GP_ERR_INVALID, "rr_pod_off or soft_pod_off does not start at 0 or decreases");
    if ((er > 0 && !r->rr_pod_name) || (es > 0 && !r->soft_pod_name)) return bad(GP_ERR_INVALID, "missing arrays or negative sizes");
    if (er + es > ((int64_t)1 << 30)) return bad(GP_ERR_INVALID, "more than 2^30 reservation entries");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t P = (size_t)p->n_pods, N = (size_t)n_nodes, R = (size_t)r->n_rr, S = (size_t)r->n_soft;
    size_t H = 64;
    while (H < 2 * (size_t)(er + es)) H <<= 1;           // at most half full: every probe ends
    Arena ar{c->overbuf};
    const size_t o_node = ar.take(4 * P), o_req = ar.take(24 * P), o_listed = ar.take(P), o_ak = ar.take(4 * P), o_ai = ar.take(4 * P),
                 o_name = ar.take(4 * P), o_exe = ar.take(P), o_spark = ar.take(P), o_has = ar.take(P),
                 o_rkey = ar.take(4 * R), o_roff = ar.take(8 * (R + 1)), o_rname = ar.take(4 * (size_t)er),
                 o_skey = ar.take(4 * S), o_soff = ar.take(8 * (S + 1)), o_sname = ar.take(4 * (size_t)es), o_qn = ar.take(4 * N),
                 o_rok = ar.take(4 * (size_t)p->n_app_keys), o_soa = ar.take(4 * (size_t)p->n_app_ids),
                 o_ron = ar.take(4 * (size_t)p->n_node_ids), o_set = ar.take(8 * H),
                 o_acc = ar.take(96 * N), o_word = ar.take(16), o_out = ar.take(48 * N);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    // the directories and the hash set start at -1 / empty; the sums, n_warned and the error word at 0
    GP_CUDA(c, cudaMemsetAsync(b + o_rok, 0xff, o_set + 8 * H - o_rok, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_acc, 0, o_word + 16 - o_acc, st));
    struct Piece { size_t o; const void* src; size_t bytes; };
    const Piece pieces[] = {
        {o_node, p->node_id, 4 * P}, {o_req, p->req_cpu_milli, 8 * P}, {o_req + 8 * P, p->req_mem_bytes, 8 * P},
        {o_req + 16 * P, p->req_gpu, 8 * P}, {o_listed, p->listed, P}, {o_ak, p->app_key, 4 * P}, {o_ai, p->app_id, 4 * P},
        {o_name, p->name_id, 4 * P}, {o_exe, p->is_executor, P}, {o_spark, p->spark_scheduler, P},
        {o_rkey, r->rr_app_key, 4 * R}, {o_roff, r->rr_pod_off, R ? 8 * (R + 1) : 0}, {o_rname, r->rr_pod_name, 4 * (size_t)er},
        {o_skey, r->soft_app_id, 4 * S}, {o_soff, r->soft_pod_off, S ? 8 * (S + 1) : 0}, {o_sname, r->soft_pod_name, 4 * (size_t)es},
        {o_qn, node_ids, 4 * N}};
    for (const Piece& pc : pieces)
        if (pc.src && pc.bytes) GP_CUDA(c, ar.upload(pc.o, pc.src, pc.bytes, st));
    OhMaps M{(int32_t*)(b + o_rok), (int32_t*)(b + o_soa), (int32_t*)(b + o_ron), (unsigned long long*)(b + o_set), (uint32_t)(H - 1),
             r->n_rr};
    int* d_err = (int*)(b + o_word + 8);
    const int T = 256, cap = c->sm_count * 8;
    const long long n_dir = (long long)R + (long long)S + (long long)N;
    if (n_dir > 0) {
        OhDirIn D{r->n_rr, r->n_soft, n_nodes, p->n_app_keys, p->n_app_ids, p->n_node_ids,
                  (const int32_t*)(b + o_rkey), (const int32_t*)(b + o_skey), (const int32_t*)(b + o_qn)};
        gp_oh_dir<<<(unsigned)std::min<long long>((n_dir + T - 1) / T, cap), T, 0, st>>>(D, M, d_err);
    }
    if (er + es > 0) {
        OhSetIn si{(const long long*)(b + o_roff), (const int32_t*)(b + o_rname), (const long long*)(b + o_soff),
                   (const int32_t*)(b + o_sname), r->n_rr, r->n_soft, p->n_names, (long long)er, (long long)es};
        gp_oh_insert<<<(unsigned)std::min<long long>((er + es + T - 1) / T, cap), T, 0, st>>>(si, M, d_err);
    }
    OhAcc A{(unsigned long long*)(b + o_acc), (unsigned long long*)(b + o_word), n_nodes};
    if (P > 0) {
        OhPodsIn pi{};
        pi.n = (long long)P; pi.n_node_ids = p->n_node_ids; pi.n_app_keys = p->n_app_keys; pi.n_app_ids = p->n_app_ids; pi.n_names = p->n_names;
        pi.node_id = (const int32_t*)(b + o_node);
        for (int d = 0; d < 3; ++d) pi.req[d] = (d < 2 || p->req_gpu) ? (const long long*)(b + o_req) + P * (size_t)d : nullptr;
        pi.listed = p->listed ? (const uint8_t*)(b + o_listed) : nullptr;
        pi.app_key = (const int32_t*)(b + o_ak); pi.app_id = (const int32_t*)(b + o_ai); pi.name_id = (const int32_t*)(b + o_name);
        pi.is_executor = p->is_executor ? (const uint8_t*)(b + o_exe) : nullptr;
        pi.spark_scheduler = p->spark_scheduler ? (const uint8_t*)(b + o_spark) : nullptr;
        pi.has_reservation = (uint8_t*)(b + o_has);
        gp_oh_pods<<<(unsigned)((P + kOhThreads - 1) / kOhThreads), kOhThreads, 0, st>>>(pi, M, A, d_err);
    }
    long long* d_out = (long long*)(b + o_out);
    if (N > 0) gp_oh_finish<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(A, d_out, d_err);
    GP_CUDA(c, cudaGetLastError());
    int64_t* outs[6] = {out->overhead_cpu_milli, out->overhead_mem_bytes, out->overhead_gpu,
                        out->nonsched_cpu_milli, out->nonsched_mem_bytes, out->nonsched_gpu};
    for (int k = 0; k < 6; ++k)
        if (outs[k] && N) GP_CUDA(c, cudaMemcpyAsync(outs[k], d_out + N * (size_t)k, 8 * N, cudaMemcpyDeviceToHost, st));
    if (out->has_reservation && P) GP_CUDA(c, cudaMemcpyAsync(out->has_reservation, b + o_has, P, cudaMemcpyDeviceToHost, st));
    unsigned long long word[2] = {0, 0};                 // n_warned, error bits
    GP_CUDA(c, cudaMemcpyAsync(word, b + o_word, 16, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    const int herr = (int)word[1];
    if (herr & kOhErrRange) return bad(GP_ERR_INVALID, "an id out of its range (node, app key, app id, name or query node)");
    if (herr & kOhErrAppPair) return bad(GP_ERR_INVALID, "app_key and app_id disagree on -1");
    if (herr & kOhErrDuplicate) return bad(GP_ERR_INVALID, "a query node id, rr_app_key or soft_app_id given twice");
    if (herr & kOhErrNegative) return bad(GP_ERR_INVALID, "negative request");
    if (herr & kOhErrRequest) return bad(GP_ERR_UNREPRESENTABLE, "request >= 2^61");
    if (herr & kOhErrSum) return bad(GP_ERR_UNREPRESENTABLE, "a per-node sum >= 2^61");
    if (out->n_warned) *out->n_warned = (int64_t)word[0];
    return GP_OK;
}

}  // extern "C"
