// gangpack_overhead_table.cu -- the resident overhead table: gp_overhead_table_reset, gp_overhead_table_update and
// gp_overhead_table_query.  The kernels are in gangpack_overhead.cuh, next to the per-call ones they share.  An update runs
// within the protocol of gangpack_resident.cuh, with the member set's rehash target staged before it starts.
#include "gangpack_ctx.cuh"
#include "gangpack_overhead.cuh"

#include <algorithm>

// Cells of the member set after a reset.  An update that could take the cells holding a key or a tombstone past half of the
// set first rehashes the live keys into max(cells, the least power of two >= 4 * (live keys + insertions)) cells.
static constexpr uint32_t kOhtInitialCells = 1024;
static constexpr long long kOhtMaxKeys = 1ll << 29;        // 4 * keys stays within the 32-bit cell index

struct OhtPieces {
    Piece<int32_t> node;
    Piece<long long> req;
    Piece<uint8_t> listed;
    Piece<int32_t> ak, ai, nm;
    Piece<uint8_t> exe, spark, rr;
    Piece<uint32_t> slot_stamp, rr_stamp;
};

// The layout of the table's column block; node first (0xff: free), everything after it starts at 0
static OhtPieces take_cols(Arena& a, const gp_overhead_table_size& z) {
    const size_t S = (size_t)z.n_slots;
    OhtPieces p;
    p.node = a.take<int32_t>(S);
    p.req = a.take<long long>(3 * S);
    p.listed = a.take<uint8_t>(S);
    p.ak = a.take<int32_t>(S); p.ai = a.take<int32_t>(S); p.nm = a.take<int32_t>(S);
    p.exe = a.take<uint8_t>(S); p.spark = a.take<uint8_t>(S);
    p.rr = a.take<uint8_t>((size_t)z.n_app_keys);
    p.slot_stamp = a.take<uint32_t>(S);
    p.rr_stamp = a.take<uint32_t>((size_t)z.n_app_keys);
    return p;
}

static OhtCols cols_of(const Arena& a, const OhtPieces& p, size_t S) {
    OhtCols T{};
    T.node_id = a.ptr(p.node);
    for (int d = 0; d < 3; ++d) T.req[d] = a.ptr(p.req.part(S * d, S));
    T.listed = a.ptr(p.listed);
    T.app_key = a.ptr(p.ak); T.app_id = a.ptr(p.ai); T.name_id = a.ptr(p.nm);
    T.is_executor = a.ptr(p.exe); T.spark_scheduler = a.ptr(p.spark);
    T.rr = a.ptr(p.rr);
    return T;
}

static const Refusal kOhtRefusals[] = {
    {kOhtErrRange, GP_ERR_INVALID, "a slot, id or member kind out of its range"},
    {kOhtErrDuplicate, GP_ERR_INVALID, "a slot, rr_app_key or member triple given twice"},
    {kOhtErrAppPair, GP_ERR_INVALID, "app_key and app_id disagree on -1"},
    {kOhtErrNegative, GP_ERR_INVALID, "negative request"},
    {kOhtErrRequest, GP_ERR_UNREPRESENTABLE, "request >= 2^61"},
};

// The rows were checked when they were written, so only the query's own inputs and the sums can be refused
static const Refusal kOhtQueryRefusals[] = {
    {kOhErrRange, GP_ERR_INVALID, "a query node id out of range"},
    {kOhErrDuplicate, GP_ERR_INVALID, "a query node id given twice"},
    {kOhErrSum, GP_ERR_UNREPRESENTABLE, "a per-node sum >= 2^61"},
};

static uint32_t pow2_at_least(long long n, uint32_t lo) {
    uint32_t h = lo;
    while ((long long)h < n) h <<= 1;
    return h;
}

void oht_enqueue_sums(gp_ctx* c, cudaStream_t st, const int32_t* row_of_node, int32_t n_rows, unsigned long long* acc,
                      unsigned long long* n_warned, long long* out, uint8_t* has_reservation, int* d_err) {
    auto& t = c->oht;
    const size_t S = (size_t)t.size.n_slots;
    Arena tc{t.cols, st};
    const OhtPieces p = take_cols(tc, t.size);
    const OhtCols T = cols_of(tc, p, S);
    const OhAcc A{acc, n_warned, n_rows};
    if (S > 0) {
        OhPodsIn pi{};
        pi.n = (long long)S;
        pi.n_node_ids = t.size.n_node_ids; pi.n_app_keys = t.size.n_app_keys; pi.n_app_ids = t.size.n_app_ids; pi.n_names = t.size.n_names;
        pi.node_id = T.node_id;
        for (int d = 0; d < 3; ++d) pi.req[d] = T.req[d];
        pi.listed = T.listed;
        pi.app_key = T.app_key; pi.app_id = T.app_id; pi.name_id = T.name_id;
        pi.is_executor = T.is_executor; pi.spark_scheduler = T.spark_scheduler;
        pi.has_reservation = has_reservation;
        const OhTableLookup L{T.rr, OhtSet{t.set[t.cur].as<unsigned long long>(), t.cells - 1}, row_of_node};
        gp_oh_pods<<<(unsigned)((S + kOhThreads - 1) / kOhThreads), kOhThreads, 0, st>>>(pi, L, A, d_err);
    }
    const int B = 256;
    if (n_rows > 0) gp_oh_finish<<<(unsigned)((n_rows + B - 1) / B), B, 0, st>>>(A, out, d_err);
}

gp_status oht_sum_refusal(gp_ctx* c, int word, const char* who) { return refuse(c, word, kOhtQueryRefusals, who); }

extern "C" {

gp_status gp_overhead_table_reset(gp_ctx* c, const gp_overhead_table_size* z) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_overhead_table_reset";
    if (!z || z->n_slots < 0 || z->n_node_ids < 0 || z->n_app_keys < 0 || z->n_app_ids < 0 || z->n_names < 0)
        return fail(c, GP_ERR_INVALID, who, "NULL size or a negative capacity");
    if (z->n_slots > INT32_MAX) return fail(c, GP_ERR_INVALID, who, "n_slots must be below 2^31");
    auto& t = c->oht;
    return t.reset(c, *z, [&](Arena& a) {
        const OhtPieces p = take_cols(a, *z);
        a.reserve();
        a.fill(p.node, 0xff);
        a.fill(p.req, p.rr_stamp, 0);
        Arena s{t.set[t.cur], a.st};
        const auto cells = s.take<unsigned long long>(kOhtInitialCells);
        s.reserve();
        s.fill(cells, 0xff);
        t.cells = kOhtInitialCells;
        t.keys = t.used = 0;
        return s.check(c);
    });
}

gp_status gp_overhead_table_update(gp_ctx* c, const gp_overhead_delta* d) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_overhead_table_update";
    auto& t = c->oht;
    GP_TRY(require(c, t.need(), who));
    if (!d || d->n_write < 0 || d->n_rr < 0 || d->n_member < 0 ||
        (d->n_write > 0 && (!d->slot || !d->node_id || !d->req_cpu_milli || !d->req_mem_bytes || !d->app_key || !d->app_id || !d->name_id)) ||
        (d->n_rr > 0 && (!d->rr_app_key || !d->rr_exists)) ||
        (d->n_member > 0 && (!d->member_kind || !d->member_app || !d->member_name || !d->member_present)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or negative counts");
    if (d->n_write > t.size.n_slots || d->n_rr > t.size.n_app_keys)
        return fail(c, GP_ERR_INVALID, who, "more slot writes than slots or RR flag writes than app keys: a slot or rr_app_key "
                                            "given twice or out of its range");
    if (d->n_member > kOhtMaxKeys) return fail(c, GP_ERR_CAPACITY, who, "more than 2^29 members");
    long long ins = 0;
    for (int64_t m = 0; m < d->n_member; ++m) ins += d->member_present[m] != 0;
    if (t.keys + ins > kOhtMaxKeys) return fail(c, GP_ERR_CAPACITY, who, "more than 2^29 members");
    const bool rehash = 2 * (t.used + ins) > (long long)t.cells;
    const uint32_t cells = rehash ? std::max(t.cells, pow2_at_least(4 * (t.keys + ins), kOhtInitialCells)) : t.cells;

    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t W = (size_t)d->n_write, R = (size_t)d->n_rr, M = (size_t)d->n_member, S = (size_t)t.size.n_slots;
    const uint32_t dup_cells = pow2_at_least(2 * (long long)M, 64);
    Arena ar{c->callbuf, st};
    const auto slot = ar.take<int32_t>(W), node = ar.take<int32_t>(W);
    const auto req = ar.take<long long>(3 * W);
    const auto listed = ar.take<uint8_t>(W);
    const auto ak = ar.take<int32_t>(W), ai = ar.take<int32_t>(W), nm = ar.take<int32_t>(W);
    const auto exe = ar.take<uint8_t>(W), spark = ar.take<uint8_t>(W);
    const auto rkey = ar.take<int32_t>(R);
    const auto rflag = ar.take<uint8_t>(R);
    const auto mkind = ar.take<uint8_t>(M);
    const auto mapp = ar.take<int32_t>(M), mname = ar.take<int32_t>(M);
    const auto mpres = ar.take<uint8_t>(M);
    const auto dup = ar.take<unsigned long long>(dup_cells);
    const auto word = ar.take<OhtWord>(1);
    ar.reserve();
    ar.fill(dup, 0xff);
    ar.zero(word);
    OhtDelta D{};
    D.n_write = (long long)W; D.n_rr = d->n_rr; D.n_member = (long long)M;
    D.n_slots = (int32_t)t.size.n_slots; D.n_node_ids = t.size.n_node_ids; D.n_app_keys = t.size.n_app_keys;
    D.n_app_ids = t.size.n_app_ids; D.n_names = t.size.n_names;
    D.slot = ar.put(slot, d->slot);
    D.node_id = ar.put(node, d->node_id);
    const int64_t* reqs[3] = {d->req_cpu_milli, d->req_mem_bytes, d->req_gpu};
    for (int k = 0; k < 3; ++k) D.req[k] = ar.put(req.part(W * k, W), reqs[k]);
    D.listed = ar.put(listed, d->listed);
    D.app_key = ar.put(ak, d->app_key); D.app_id = ar.put(ai, d->app_id); D.name_id = ar.put(nm, d->name_id);
    D.is_executor = ar.put(exe, d->is_executor);
    D.spark_scheduler = ar.put(spark, d->spark_scheduler);
    D.rr_app_key = ar.put(rkey, d->rr_app_key);
    D.rr_exists = ar.put(rflag, d->rr_exists);
    D.member_kind = ar.put(mkind, d->member_kind);
    D.member_app = ar.put(mapp, d->member_app); D.member_name = ar.put(mname, d->member_name);
    D.member_present = ar.put(mpres, d->member_present);
    GP_TRY(ar.check(c));
    // the rehash target is the spare set, not the live one: staging it, like the delta, writes nothing the table holds
    Arena nx{t.set[t.cur ^ 1], st};
    const auto to = nx.take<unsigned long long>(rehash ? cells : 0);
    if (rehash) {
        nx.reserve();
        nx.fill(to, 0xff);
        GP_TRY(nx.check(c));
    }
    Arena tc{t.cols, st};
    const OhtPieces p = take_cols(tc, t.size);
    GP_TRY(t.begin(c, tc, p.slot_stamp, p.rr_stamp));
    OhtWord* w = ar.ptr(word);
    const int T = 256;
    auto grid = [&](long long n) { return update_grid(n, T, c->sm_count); };
    const long long total = (long long)W + (long long)R + (long long)M;
    if (total > 0)
        gp_oht_check<<<grid(total), T, 0, st>>>(D, tc.ptr(p.slot_stamp), tc.ptr(p.rr_stamp), t.seq, OhtSet{ar.ptr(dup), dup_cells - 1}, w);
    OhtSet set{t.set[t.cur].as<unsigned long long>(), t.cells - 1};
    if (rehash) {                                            // the same keys in a fresh set, whatever the delta's verdict
        const OhtSet next{nx.ptr(to), cells - 1};
        gp_oht_rehash<<<grid((long long)t.cells), T, 0, st>>>(set, next);
        set = next;
        t.cur ^= 1;
        t.cells = cells;
        t.used = t.keys;
    }
    if (total > 0) gp_oht_apply<<<grid(total), T, 0, st>>>(D, cols_of(tc, p, S), set, w);
    if (ins > 0) gp_oht_insert<<<grid((long long)M), T, 0, st>>>(D, set, w);
    OhtWord hw{};
    GP_TRY(t.commit(c, ar, word, &hw, kOhtRefusals, who));
    t.keys += (long long)hw.inserted - (long long)hw.removed;
    t.used += (long long)hw.inserted;
    return GP_OK;
}

gp_status gp_overhead_table_query(gp_ctx* c, int32_t n_nodes, const int32_t* node_ids, gp_overhead_out* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_overhead_table_query";
    auto& t = c->oht;
    GP_TRY(require(c, t.need(), who));
    if (!out || n_nodes < 0 || (n_nodes > 0 && !node_ids)) return fail(c, GP_ERR_INVALID, who, "missing arrays or negative sizes");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t N = (size_t)n_nodes, S = (size_t)t.size.n_slots;
    struct OhWord { unsigned long long n_warned; int err, unused; };
    Arena ar{c->callbuf, st};
    const auto qn = ar.take<int32_t>(N);
    const auto ron = ar.take<int32_t>((size_t)t.size.n_node_ids);
    const auto acc = ar.take<unsigned long long>(12 * N);
    const auto word = ar.take<OhWord>(1);
    const auto d_out = ar.take<long long>(6 * N);
    const auto has = ar.take<uint8_t>(out->has_reservation ? S : 0);
    ar.reserve();
    ar.fill(ron, 0xff);
    ar.fill(acc, word, 0);
    ar.put(qn, node_ids);
    GP_TRY(ar.check(c));
    int* d_err = &ar.ptr(word)->err;
    const int B = 256, cap = c->sm_count * 8;
    OhMaps M{nullptr, nullptr, ar.ptr(ron), nullptr, 0, 0};
    if (N > 0) {
        OhDirIn D{0, 0, n_nodes, 0, 0, t.size.n_node_ids, nullptr, nullptr, ar.ptr(qn)};
        gp_oh_dir<<<(unsigned)std::min<long long>(((long long)N + B - 1) / B, cap), B, 0, st>>>(D, M, d_err);
    }
    oht_enqueue_sums(c, st, ar.ptr(ron), n_nodes, ar.ptr(acc), &ar.ptr(word)->n_warned, ar.ptr(d_out),
                     out->has_reservation ? ar.ptr(has) : nullptr, d_err);
    GP_CUDA(c, cudaGetLastError());
    int64_t* outs[6] = {out->overhead_cpu_milli, out->overhead_mem_bytes, out->overhead_gpu,
                        out->nonsched_cpu_milli, out->nonsched_mem_bytes, out->nonsched_gpu};
    for (int k = 0; k < 6; ++k) ar.get(outs[k], d_out.part(N * k, N));
    ar.get(out->has_reservation, has);
    OhWord hw{};
    ar.get(&hw, word);
    GP_TRY(ar.sync(c));
    GP_TRY(refuse(c, hw.err, kOhtQueryRefusals, who));
    if (out->n_warned) *out->n_warned = (int64_t)hw.n_warned;
    return GP_OK;
}

}  // extern "C"
