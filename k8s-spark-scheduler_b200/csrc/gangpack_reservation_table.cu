// gangpack_reservation_table.cu -- the resident reservation table: gp_reservation_table_reset and gp_reservation_table_update.
// The *_resident entries of gangpack_cluster.cu read it through rt_cols().
//
// An update runs
//   gp_rt_check   thread per write: slot and node id ranges, duplicate slots (stamped_twice), |value| < 2^61; sets the error
//                 word and writes nothing but the stamps
//   gp_rt_apply   thread per write: the whole row; nothing when the error word is set
// within the update protocol of gangpack_resident.cuh, so a refused delta leaves the table as it was.
#include "gangpack_ctx.cuh"

enum : int {
    kRtErrRange = 1,            // a slot or node id out of its range
    kRtErrDuplicate = 2,        // a slot given twice
    kRtErrValue = 4,            // |cpu|, |mem| or |gpu| >= 2^61 on an occupied row
};

static const Refusal kRtRefusals[] = {
    {kRtErrRange, GP_ERR_INVALID, "a slot or node id out of its range"},
    {kRtErrDuplicate, GP_ERR_INVALID, "a slot given twice"},
    {kRtErrValue, GP_ERR_UNREPRESENTABLE, "|reservation| >= 2^61"},
};

struct RtPieces {
    Piece<int32_t> node;
    Piece<long long> v;
    Piece<uint32_t> stamp;
};

// The layout of the table's column block: node ids first (0xff: free), then the values and the stamps (0)
static RtPieces take_cols(Arena& a, const gp_reservation_table_size& z) {
    const size_t S = (size_t)z.n_slots;
    RtPieces p;
    p.node = a.take<int32_t>(S);
    p.v = a.take<long long>(3 * S);
    p.stamp = a.take<uint32_t>(S);
    return p;
}

// One update, staged on the device; gpu NULL = 0
struct RtDelta {
    long long n;
    int32_t n_slots, n_node_ids;
    const int32_t* slot;
    const int32_t* node_id;
    const long long* v[3];
};

__global__ void gp_rt_check(RtDelta D, uint32_t* __restrict__ stamp, uint32_t seq, int* __restrict__ err) {
    int bad = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < D.n; i += (long long)gridDim.x * blockDim.x) {
        const int32_t s = D.slot[i], node = D.node_id[i];
        if (s < 0 || s >= D.n_slots) { bad |= kRtErrRange; continue; }
        if (stamped_twice(stamp + s, seq)) bad |= kRtErrDuplicate;
        if (node == -1) continue;                                      // a free slot: its values are not read
        if (node < 0 || node >= D.n_node_ids) bad |= kRtErrRange;
        for (int d = 0; d < 3; ++d) {
            const long long x = D.v[d] ? D.v[d][i] : 0;
            if (x >= kMaxQuantity || x <= -kMaxQuantity) bad |= kRtErrValue;
        }
    }
    if (bad) atomicOr(err, bad);
}

__global__ void gp_rt_apply(RtDelta D, int32_t* __restrict__ node, long long* __restrict__ v, const int* __restrict__ err) {
    if (*(volatile const int*)err) return;
    const size_t S = (size_t)D.n_slots;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < D.n; i += (long long)gridDim.x * blockDim.x) {
        const int32_t s = D.slot[i], id = D.node_id[i];
        node[s] = id;
        for (int d = 0; d < 3; ++d) v[S * d + s] = id != -1 && D.v[d] ? D.v[d][i] : 0;
    }
}

RtCols rt_cols(gp_ctx* c) {
    auto& t = c->rt;
    Arena a{t.cols, c->stream};
    const RtPieces p = take_cols(a, t.size);
    const size_t S = (size_t)t.size.n_slots;
    RtCols r{a.ptr(p.node), {}};
    for (int d = 0; d < 3; ++d) r.v[d] = a.ptr(p.v.part(S * d, S));
    return r;
}

extern "C" {

gp_status gp_reservation_table_reset(gp_ctx* c, const gp_reservation_table_size* z) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_reservation_table_reset";
    if (!z || z->n_slots < 0 || z->n_node_ids < 0) return fail(c, GP_ERR_INVALID, who, "NULL size or a negative capacity");
    if (z->n_slots > INT32_MAX) return fail(c, GP_ERR_INVALID, who, "n_slots must be below 2^31");
    return c->rt.reset(c, *z, [&](Arena& a) {
        const RtPieces p = take_cols(a, *z);
        a.reserve();
        a.fill(p.node, 0xff);
        a.fill(p.v, p.stamp, 0);
        return GP_OK;
    });
}

gp_status gp_reservation_table_update(gp_ctx* c, const gp_reservation_delta* d) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_reservation_table_update";
    auto& t = c->rt;
    GP_TRY(require(c, t.need(), who));
    if (!d || d->n_write < 0 || (d->n_write > 0 && (!d->slot || !d->node_id || !d->cpu_milli || !d->mem_bytes)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative count");
    if (d->n_write > t.size.n_slots) return fail(c, GP_ERR_INVALID, who, "more slot writes than slots: a slot given twice or out of range");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t W = (size_t)d->n_write;
    Arena ar{c->callbuf, st};
    const auto slot = ar.take<int32_t>(W), node = ar.take<int32_t>(W);
    const auto val = ar.take<long long>(3 * W);
    const auto word = ar.take<int>(1);
    ar.reserve();
    ar.zero(word);
    RtDelta D{};
    D.n = (long long)W;
    D.n_slots = (int32_t)t.size.n_slots; D.n_node_ids = t.size.n_node_ids;
    D.slot = ar.put(slot, d->slot);
    D.node_id = ar.put(node, d->node_id);
    const int64_t* vals[3] = {d->cpu_milli, d->mem_bytes, d->gpu};
    for (int k = 0; k < 3; ++k) D.v[k] = ar.put(val.part(W * k, W), vals[k]);
    GP_TRY(ar.check(c));
    Arena tc{t.cols, st};
    const RtPieces p = take_cols(tc, t.size);
    GP_TRY(t.begin(c, tc, p.stamp, p.stamp));
    int* w = ar.ptr(word);
    if (W > 0) {
        const int T = 256;
        const unsigned grid = update_grid((long long)W, T, c->sm_count);
        gp_rt_check<<<grid, T, 0, st>>>(D, tc.ptr(p.stamp), t.seq, w);
        gp_rt_apply<<<grid, T, 0, st>>>(D, tc.ptr(p.node), tc.ptr(p.v), w);
    }
    int hw = 0;
    return t.commit(c, ar, word, &hw, kRtRefusals, who);
}

}  // extern "C"
