// gangpack_label_table.cu -- the resident label table: gp_label_table_reset and gp_label_table_update.  The resident affinity
// entries of gangpack_marker.cu read it through lt_cols() as gp_aff_match's AffLabelsResident source.
//
// An update runs
//   gp_lt_check   thread per row write and per value write: node and value id ranges, duplicates (per-row and per-value
//                 stamps, stamped_twice), row length within the stride, key ids in range and strictly ascending, label value
//                 ids in range; sets the error word and writes nothing but the stamps
//   gp_lt_apply   the same threads: the whole row (count, keys, values) or the value's ParseInt columns; nothing when the
//                 error word is set
// within the update protocol of gangpack_resident.cuh, so a refused delta leaves the table as it was.
#include "gangpack_ctx.cuh"

enum : int {
    kLtErrRange = 1,            // a node or value id out of its range
    kLtErrDuplicate = 2,        // a node or value id given twice
    kLtErrLength = 4,           // a row longer than max_labels
    kLtErrKey = 8,              // a key id out of range, or the keys of a row not strictly ascending
    kLtErrValue = 16,           // a label value id out of range
};

static const Refusal kLtRefusals[] = {
    {kLtErrRange, GP_ERR_INVALID, "a node or value id out of its range"},
    {kLtErrDuplicate, GP_ERR_INVALID, "a node or value id given twice"},
    {kLtErrLength, GP_ERR_INVALID, "a row longer than max_labels"},
    {kLtErrKey, GP_ERR_INVALID, "a label key id out of range or the keys of a row not strictly ascending"},
    {kLtErrValue, GP_ERR_INVALID, "a label value id out of range"},
};

struct LtPieces {
    Piece<int32_t> count, key, val;
    Piece<long long> vint;
    Piece<uint8_t> vok;
    Piece<uint32_t> rstamp, vstamp;
};

// The layout of the table's column block: counts, the two stride columns, then the value columns and the stamps (all 0 after
// a reset; the stride columns are read only below each row's count)
static LtPieces take_cols(Arena& a, const gp_label_table_size& z) {
    const size_t R = (size_t)z.n_node_ids, V = (size_t)z.n_values, E = R * (size_t)z.max_labels;
    LtPieces p;
    p.count = a.take<int32_t>(R);
    p.key = a.take<int32_t>(E);
    p.val = a.take<int32_t>(E);
    p.vint = a.take<long long>(V);
    p.vok = a.take<uint8_t>(V);
    p.rstamp = a.take<uint32_t>(R);
    p.vstamp = a.take<uint32_t>(V);
    return p;
}

// One update, staged on the device: items [0, n_rows) are row writes, [n_rows, n_rows + n_vals) value writes
struct LtDelta {
    int32_t n_rows, n_vals;
    int32_t n_node_ids, stride, n_keys, n_values;
    const int32_t* row_node;
    const long long* row_off;
    const int32_t* key;
    const int32_t* val;
    const int32_t* value_id;
    const uint8_t* int_ok;
    const long long* ival;
};

__global__ void gp_lt_check(LtDelta D, uint32_t* __restrict__ rstamp, uint32_t* __restrict__ vstamp, uint32_t seq, int* __restrict__ err) {
    int bad = 0;
    const long long total = (long long)D.n_rows + D.n_vals;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < D.n_rows) {
            const int32_t r = D.row_node[i];
            if (r < 0 || r >= D.n_node_ids) { bad |= kLtErrRange; continue; }
            if (stamped_twice(rstamp + r, seq)) bad |= kLtErrDuplicate;
            const long long lo = D.row_off[i], hi = D.row_off[i + 1];
            if (hi - lo > D.stride) { bad |= kLtErrLength; continue; }
            for (long long e = lo; e < hi; ++e) {
                const int32_t k = D.key[e], v = D.val[e];
                if (k < 0 || k >= D.n_keys || (e > lo && k <= D.key[e - 1])) bad |= kLtErrKey;
                if (v < 0 || v >= D.n_values) bad |= kLtErrValue;
            }
        } else {
            const int32_t v = D.value_id[i - D.n_rows];
            if (v < 0 || v >= D.n_values) { bad |= kLtErrRange; continue; }
            if (stamped_twice(vstamp + v, seq)) bad |= kLtErrDuplicate;
        }
    }
    if (bad) atomicOr(err, bad);
}

__global__ void gp_lt_apply(LtDelta D, int32_t* __restrict__ count, int32_t* __restrict__ key, int32_t* __restrict__ val,
                            long long* __restrict__ vint, uint8_t* __restrict__ vok, const int* __restrict__ err) {
    if (*(volatile const int*)err) return;
    const long long total = (long long)D.n_rows + D.n_vals;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < D.n_rows) {
            const int32_t r = D.row_node[i];
            const long long lo = D.row_off[i], hi = D.row_off[i + 1], base = (long long)r * D.stride - lo;
            count[r] = (int32_t)(hi - lo);
            for (long long e = lo; e < hi; ++e) { key[base + e] = D.key[e]; val[base + e] = D.val[e]; }
        } else {
            const long long j = i - D.n_rows;
            const int32_t v = D.value_id[j];
            const bool ok = D.int_ok[j] != 0;
            vok[v] = ok ? 1 : 0;
            vint[v] = ok ? D.ival[j] : 0;
        }
    }
}

LtCols lt_cols(gp_ctx* c) {
    auto& t = c->lt;
    Arena a{t.cols, c->stream};
    const LtPieces p = take_cols(a, t.size);
    return {a.ptr(p.count), a.ptr(p.key), a.ptr(p.val), a.ptr(p.vint), a.ptr(p.vok)};
}

extern "C" {

gp_status gp_label_table_reset(gp_ctx* c, const gp_label_table_size* z) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_label_table_reset";
    if (!z || z->n_node_ids < 0 || z->max_labels < 0 || z->n_keys < 0 || z->n_values < 0)
        return fail(c, GP_ERR_INVALID, who, "NULL size or a negative capacity");
    if ((int64_t)z->n_node_ids * z->max_labels > INT32_MAX) return fail(c, GP_ERR_INVALID, who, "n_node_ids * max_labels must be below 2^31");
    return c->lt.reset(c, *z, [&](Arena& a) {
        const LtPieces p = take_cols(a, *z);
        a.reserve();
        a.zero(p.count);
        a.fill(p.vint, p.vstamp, 0);
        return GP_OK;
    });
}

gp_status gp_label_table_update(gp_ctx* c, const gp_label_delta* d) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_label_table_update";
    auto& t = c->lt;
    GP_TRY(require(c, t.need(), who));
    if (!d || d->n_rows < 0 || d->n_values < 0 || (d->n_rows > 0 && (!d->row_node || !d->row_off)) ||
        (d->n_values > 0 && (!d->value_id || !d->value_int_ok || !d->value_int)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative count");
    int64_t P = 0;
    if (d->n_rows > 0) {                                     // CSR offsets (host-sized); the entries are checked on the device
        if (d->row_off[0] != 0) return fail(c, GP_ERR_INVALID, who, "row_off does not start at 0 or decreases");
        for (int32_t i = 0; i < d->n_rows; ++i)
            if (d->row_off[i + 1] < d->row_off[i]) return fail(c, GP_ERR_INVALID, who, "row_off does not start at 0 or decreases");
        P = d->row_off[d->n_rows];
        if (P > 0 && (!d->label_key || !d->label_val)) return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative count");
    }
    if (d->n_rows > t.size.n_node_ids || d->n_values > t.size.n_values)
        return fail(c, GP_ERR_INVALID, who, "more writes than ids: a node or value id given twice or out of range");
    if (P > (int64_t)d->n_rows * t.size.max_labels) return fail(c, GP_ERR_INVALID, who, "a row longer than max_labels");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t Rw = (size_t)d->n_rows, Vw = (size_t)d->n_values;
    Arena ar{c->callbuf, st};
    const auto rnode = ar.take<int32_t>(Rw);
    const auto roff = ar.take<long long>(Rw ? Rw + 1 : 0);
    const auto key = ar.take<int32_t>((size_t)P), val = ar.take<int32_t>((size_t)P);
    const auto vid = ar.take<int32_t>(Vw);
    const auto vok = ar.take<uint8_t>(Vw);
    const auto vint = ar.take<long long>(Vw);
    const auto word = ar.take<int>(1);
    ar.reserve();
    ar.zero(word);
    LtDelta D{};
    D.n_rows = d->n_rows; D.n_vals = d->n_values;
    D.n_node_ids = t.size.n_node_ids; D.stride = t.size.max_labels; D.n_keys = t.size.n_keys; D.n_values = t.size.n_values;
    D.row_node = ar.put(rnode, d->row_node);
    D.row_off = Rw ? ar.put(roff, d->row_off) : nullptr;
    D.key = ar.put(key, d->label_key);
    D.val = ar.put(val, d->label_val);
    D.value_id = ar.put(vid, d->value_id);
    D.int_ok = ar.put(vok, d->value_int_ok);
    D.ival = ar.put(vint, d->value_int);
    GP_TRY(ar.check(c));
    Arena tc{t.cols, st};
    const LtPieces p = take_cols(tc, t.size);
    GP_TRY(t.begin(c, tc, p.rstamp, p.vstamp));
    int* w = ar.ptr(word);
    const long long items = (long long)Rw + (long long)Vw;
    if (items > 0) {
        const int T = 256;
        const unsigned grid = update_grid(items, T, c->sm_count);
        gp_lt_check<<<grid, T, 0, st>>>(D, tc.ptr(p.rstamp), tc.ptr(p.vstamp), t.seq, w);
        gp_lt_apply<<<grid, T, 0, st>>>(D, tc.ptr(p.count), tc.ptr(p.key), tc.ptr(p.val), tc.ptr(p.vint), tc.ptr(p.vok), w);
    }
    int hw = 0;
    return t.commit(c, ar, word, &hw, kLtRefusals, who);
}

}  // extern "C"
