// gangpack_driver_table.cu -- the resident driver table: gp_driver_table_reset and gp_driver_table_update, and the two entries
// that select, order and pack a FIFO queue from it (gp_pack_fifo_driver_table, gp_pack_fifo_zones_groups_driver_table).
//
// An update runs
//   gp_dt_check     thread per slot write: slot range, duplicates (per-slot stamps, stamped_twice), on present rows scheduler
//                   and group range and |quantity| < 2^61 when the row is exact
//   gp_dt_apply     the slot writes; nothing when the error word is set
//   gp_dt_apply_aff the affinity column's writes, under the same error word
// within the update protocol of gangpack_resident.cuh, so a refused delta leaves the table as it was.
//
// The queue stage of an entry writes, on the device, exactly the gp_apps columns the host would upload for the same pods
// (filterToEarliestAndSort stable in slot order, sparkResources, shouldSkipDriverFifo):
//   gp_dq_select    thread per slot: the rows the query selects, compacted (warp ballot, block scan, one atomicAdd per
//                   block) into QueueKeys (snapshot group, creation, slot); a selected inexact row or an absent requesting
//                   row sets the refusal word
//   gp_sort_tiles / gp_rank_by_search <QueueKey>   pos[i] = the queue position of compacted row i (count on the device)
//   gp_dq_scatter   thread per queued row: its slot, six quantities, count, snapshot group, skip flag and creation at its
//                   position; the Predicate form's requesting row after them
//   gp_dq_finish    one CTA: the exclusive scan of max(count, 0) (the ExecutorNodes offsets), the undefined ties, and for the
//                   zone drain the per-instance-group counts and largest count and the identity queue
// then one synchronise reads the count, the executor total and the refusal word, so every refusal comes before any pack
// launch.  The existing FIFO bodies then run unchanged on these device columns: pack_begin + pack_device_range as
// gp_pack_batch_device runs them, or fifo_zones_body (gangpack_zones.cu) in place of its upload.
//
// The unschedulable-pod marker's stale stage (dt_stale_stage, for gp_exceeds_cluster_capacity_driver_table) has the same shape:
//   gp_ds_select    thread per slot: present, the swept scheduler and creation + timeout < now (exact, 128 bits), compacted
//                   into QueueKeys (0, creation, slot) by the same block compaction; an affinity id outside [-1, n_aff) on a
//                   stale row sets the refusal word
//   gp_sort_tiles / gp_rank_by_search <QueueKey>   the (creation, slot) order
//   gp_ds_scatter   thread per stale row: its slot, six quantities, count and capacity group (the affinity id, -1 -> n_aff) at
//                   its position, or an all-zero placeholder with outcome 2 for a row outside the model
// then one synchronise reads the count and the refusal word before the capacity kernels run on the columns.
#include "gangpack_ctx.cuh"
#include "gangpack_tilesort.cuh"

#include <algorithm>
#include <vector>

namespace gp {

// the order key of a queued row: (snapshot group, creation, slot) in 16 bytes.  A tile of 4 096 is 64 KB of dynamic shared
// memory, above the default 48 KB: gp_sort_tiles<QueueKey> is opted in with cudaFuncSetAttribute once per device (creation
// needs its 64 bits, so the key does not pack into the node table's 12 bytes).
struct QueueKey {
    int32_t sg;
    int32_t slot;
    long long creation;
};
__device__ __forceinline__ bool key_less(const QueueKey& a, const QueueKey& b) {
    return a.sg != b.sg ? a.sg < b.sg : (a.creation != b.creation ? a.creation < b.creation : a.slot < b.slot);
}
__device__ __forceinline__ QueueKey key_max(const QueueKey*) {
    QueueKey k; k.sg = 0x7fffffff; k.slot = 0x7fffffff; k.creation = 0x7fffffffffffffffLL; return k;
}

}  // namespace gp

static_assert(sizeof(QueueKey) == 16, "QueueKey layout");

enum : int {
    kDtErrRange = 1,            // a slot out of range
    kDtErrDuplicate = 2,        // a slot given twice
    kDtErrId = 4,               // a scheduler or group id out of range on a present row
    kDtErrInput = 8,            // |quantity| >= 2^61 on an exact present row
};

static const Refusal kDtRefusals[] = {
    {kDtErrRange, GP_ERR_INVALID, "a slot out of range"},
    {kDtErrDuplicate, GP_ERR_INVALID, "a slot given twice"},
    {kDtErrId, GP_ERR_INVALID, "a scheduler outside [0, n_schedulers) or a group outside [-1, n_groups) on a present row"},
    {kDtErrInput, GP_ERR_UNREPRESENTABLE, "|quantity| >= 2^61 on a present row with exact = 1"},
};

enum : int {
    kDqErrAbsent = 1,           // the requesting slot holds no row
    kDqErrInexact = 2,          // a queued row with exact = 0
};

static const Refusal kDqRefusals[] = {
    {kDqErrAbsent, GP_ERR_INVALID, "the requesting slot holds no driver"},
    {kDqErrInexact, GP_ERR_UNREPRESENTABLE, "a queued driver has a quantity outside the exact-int64 model (exact = 0)"},
};

struct DtPieces {
    Piece<uint8_t> present, exact;
    Piece<long long> creation, q;
    Piece<int32_t> sched, group, count, aff;
    Piece<uint32_t> stamp;
};

// The layout of the table's column block (all 0 after a reset: no row present)
static DtPieces take_cols(Arena& a, const gp_driver_table_size& z) {
    const size_t S = (size_t)z.n_slots;
    DtPieces p;
    p.present = a.take<uint8_t>(S);
    p.exact = a.take<uint8_t>(S);
    p.creation = a.take<long long>(S);
    p.q = a.take<long long>(6 * S);
    p.sched = a.take<int32_t>(S);
    p.group = a.take<int32_t>(S);
    p.count = a.take<int32_t>(S);
    p.aff = a.take<int32_t>(S);
    p.stamp = a.take<uint32_t>(S);
    return p;
}

// The table's columns on the device
struct DtTable {
    uint8_t* present; uint8_t* exact;
    long long* creation;
    long long* q;                     // [6][n_slots]: drv cpu, mem, gpu, exe cpu, mem, gpu
    int32_t* sched; int32_t* group; int32_t* count;
};

static DtTable table_cols(gp_ctx* c) {
    Arena tc{c->dt.cols, c->stream};
    const DtPieces p = take_cols(tc, c->dt.size);
    return DtTable{tc.ptr(p.present), tc.ptr(p.exact), tc.ptr(p.creation), tc.ptr(p.q), tc.ptr(p.sched), tc.ptr(p.group), tc.ptr(p.count)};
}

// The affinity column [n_slots]: the marker's alone, so it stays out of DtTable (gp_dt_apply and the queue stage do not see it)
static int32_t* table_aff(gp_ctx* c) {
    Arena tc{c->dt.cols, c->stream};
    return tc.ptr(take_cols(tc, c->dt.size).aff);
}

// One update, staged on the device
struct DtDelta {
    int32_t n, n_rows, n_groups, n_sched;
    const int32_t* slot;
    const uint8_t* present;
    const long long* creation;
    const int32_t* sched;
    const int32_t* group;
    const long long* q[6];            // gpu columns NULL: 0
    const int32_t* count;
    const uint8_t* exact;
};

__global__ void gp_dt_check(DtDelta D, uint32_t* __restrict__ stamp, uint32_t seq, int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.n) return;
    const int32_t r = D.slot[i];
    if (r < 0 || r >= D.n_rows) { atomicOr(err, kDtErrRange); return; }
    int bad = stamped_twice(stamp + r, seq) ? kDtErrDuplicate : 0;
    if (D.present[i]) {
        const int32_t s = D.sched[i], g = D.group[i];
        if (s < 0 || s >= D.n_sched || g < -1 || g >= D.n_groups) bad |= kDtErrId;
        if (D.exact[i])
            for (int d = 0; d < 6; ++d)
                if (D.q[d] && (D.q[d][i] <= -kMaxQuantity || D.q[d][i] >= kMaxQuantity)) bad |= kDtErrInput;
    }
    if (bad) atomicOr(err, bad);
}

__global__ void gp_dt_apply(DtDelta D, DtTable T, const int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.n || *(volatile const int*)err) return;
    const int32_t r = D.slot[i];
    const bool on = D.present[i] != 0;
    const size_t S = (size_t)D.n_rows;
    T.present[r] = on ? 1 : 0;
    T.exact[r] = on && D.exact[i] ? 1 : 0;
    T.creation[r] = on ? D.creation[i] : 0;
    T.sched[r] = on ? D.sched[i] : 0;
    T.group[r] = on ? D.group[i] : -1;
    T.count[r] = on ? D.count[i] : 0;
    for (int d = 0; d < 6; ++d) T.q[(size_t)d * S + r] = on && D.q[d] ? D.q[d][i] : 0;
}

// the affinity ids of the same writes (aff NULL: -1), after gp_dt_apply and under its error word
__global__ void gp_dt_apply_aff(int32_t n, const int32_t* __restrict__ slot, const uint8_t* __restrict__ present,
                                const int32_t* __restrict__ aff, int32_t* __restrict__ col, const int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || *(volatile const int*)err) return;
    col[slot[i]] = present[i] && aff ? aff[i] : -1;
}

// ---- the queue stage ----

// The words the host reads after the queue stage
struct DqWords {
    int32_t selected;                 // compacted rows (the atomicAdd cursor of gp_dq_select)
    int32_t err;                      // kDqErr* bits
    int32_t n_queued;                 // selected + the requesting row
    int32_t ties;                     // undefined_ties
    long long total;                  // ExecutorNodes entries
};

struct DqIn {
    int32_t n_rows;
    int32_t req;                      // requesting slot, -1: drain form
    int32_t scheduler;                // drain form
    int32_t pred_group;               // Predicate form: the snapshot group of every entry
    const int32_t* sgmap;             // drain form: [n_groups] snapshot group of each table group
    const long long* age;             // [n_groups] enforce_after_ns
    long long now;
    const uint8_t* present; const uint8_t* exact;
    const long long* creation;
    const long long* q;               // [6][n_rows]
    const int32_t* sched; const int32_t* group; const int32_t* count;
};

// The queue columns, at queue positions; every column holds n_rows + 1 entries
struct DqOut {
    int32_t cap;                      // n_rows + 1: the column pitch of q
    int32_t* slot;
    long long* q;                     // [6][cap]
    int32_t* count; int32_t* group;
    uint8_t* skip;
    long long* creation;
    long long* off;                   // [cap + 1]
    int32_t* qidx;                    // zone drain: the identity queue, or NULL
    int32_t* gcount; int32_t* gmax;   // zone drain: [n_instance_groups] zeroed by the caller, or NULL
};

constexpr int kDqThreads = 256;

// The compacted index of this thread's entry among the selected ones of every block (meaningful where sel): a warp ballot, a
// scan of the warp counts by one thread, and one atomicAdd on *cursor per block.  Every thread of the block calls it.
template <int kThreads>
__device__ __forceinline__ int32_t block_compact(bool sel, int32_t* cursor) {
    __shared__ int32_t wsum[kThreads / 32];
    __shared__ int32_t base;
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {
        int32_t acc = 0;
        for (int k = 0; k < kThreads / 32; ++k) { const int32_t t = wsum[k]; wsum[k] = acc; acc += t; }
        base = acc ? atomicAdd(cursor, acc) : 0;
    }
    __syncthreads();
    return base + wsum[warp] + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kDqThreads) gp_dq_select(DqIn in, QueueKey* __restrict__ keys, DqWords* __restrict__ w) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    bool sel = false;
    int32_t sg = 0;
    if (r < in.n_rows && in.present[r]) {
        if (in.req >= 0) {
            const int32_t g = in.group[in.req];
            sel = g != -1 && in.group[r] == g && in.sched[r] == in.sched[in.req] && in.creation[r] < in.creation[in.req];
            sg = in.pred_group;
        } else {
            const int32_t g = in.group[r];
            sel = in.sched[r] == in.scheduler && g >= 0 && in.sgmap[g] >= 0;
            if (sel) sg = in.sgmap[g];
        }
    }
    int bad = sel && !in.exact[r] ? kDqErrInexact : 0;
    if (r == 0 && in.req >= 0) bad |= !in.present[in.req] ? kDqErrAbsent : (!in.exact[in.req] ? kDqErrInexact : 0);
    if (bad) atomicOr(&w->err, bad);
    const int32_t at = block_compact<kDqThreads>(sel, &w->selected);
    if (sel) {
        QueueKey k; k.sg = sg; k.slot = r; k.creation = in.creation[r];
        keys[at] = k;
    }
}

__global__ void gp_dq_scatter(DqIn in, const QueueKey* __restrict__ keys, const int32_t* __restrict__ pos, const DqWords* __restrict__ w,
                              DqOut o) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t n = w->selected;
    int32_t r, p, sg;
    uint8_t skip;
    if (i < n) {
        const QueueKey k = keys[i];
        r = k.slot; p = pos[i]; sg = k.sg;
        // shouldSkipDriverFifo: creation + age > now, exactly (creation > now - age in 128 bits)
        skip = (__int128)k.creation > (__int128)in.now - (__int128)in.age[in.group[r]] ? 1 : 0;
    } else if (i == n && in.req >= 0) {
        r = in.req; p = n; sg = in.pred_group; skip = 0;
    } else {
        return;
    }
    const size_t S = (size_t)in.n_rows, C = (size_t)o.cap;
    o.slot[p] = r;
    for (int d = 0; d < 6; ++d) o.q[(size_t)d * C + p] = in.q[(size_t)d * S + r];
    o.count[p] = in.count[r];
    o.group[p] = sg;
    o.skip[p] = skip;
    o.creation[p] = in.creation[r];
}

constexpr int kDqFinishThreads = 1024;

__global__ void __launch_bounds__(kDqFinishThreads) gp_dq_finish(int32_t req, DqOut o, DqWords* __restrict__ w) {
    __shared__ long long wtot[kDqFinishThreads / 32];
    __shared__ long long btot;
    __shared__ int32_t ties;
    const int32_t n = w->selected + (req >= 0 ? 1 : 0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) ties = 0;
    __syncthreads();                          // the zero is in place before any thread counts a tie
    long long carry = 0;
    for (int32_t b0 = 0; b0 < n; b0 += kDqFinishThreads) {
        const int32_t i = b0 + threadIdx.x;
        int32_t k = 0;
        if (i < n) {
            k = o.count[i];
            if (i > 0 && o.group[i] == o.group[i - 1] && o.creation[i] == o.creation[i - 1]) atomicAdd(&ties, 1);
            if (o.qidx) {
                o.qidx[i] = i;
                atomicAdd(o.gcount + o.group[i], 1);
                atomicMax(o.gmax + o.group[i], max(k, 0));
            }
        }
        // inclusive scan of max(count, 0) over the CTA: warp shuffles, then the warp totals
        long long v = max(k, 0), x = v;
        for (int d = 1; d < 32; d <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            long long t = wtot[lane], s = t;
            for (int d = 1; d < 32; d <<= 1) {
                const long long y = __shfl_up_sync(0xffffffffu, s, d);
                if (lane >= d) s += y;
            }
            wtot[lane] = s - t;               // exclusive: the warps before
            if (lane == 31) btot = s;
        }
        __syncthreads();
        const long long incl = carry + wtot[warp] + x;
        if (i < n) o.off[i] = incl - v;
        carry += btot;
        __syncthreads();                      // wtot and btot are rewritten by the next round
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        o.off[n] = carry;
        w->n_queued = n;
        w->total = carry;
        w->ties = ties;
    }
}

// What an entry packs after the queue stage: device columns of n_queued entries, and the staging arena they live in
struct QueueRun {
    int32_t n_queued;
    int64_t total;
    DqOut cols;
};

// The queue stage of both entries: host checks, the kernels, one synchronise, the refusals, and the queue_slot /
// exec_out_off downloads enqueued (completed by the pack's synchronise).  n_sg: the snapshot groups a queued row may be in;
// zones: the per-instance-group counts are wanted (c->zone_groups is filled from them).  executor_cap: the results' capacity.
static gp_status queue_stage(gp_ctx* c, const gp_driver_queue* dq, int32_t n_sg, bool zones, int64_t executor_cap, const char* who,
                             QueueRun* run) {
    auto& t = c->dt;
    GP_TRY(require(c, t.need(), who));
    const int32_t S = t.size.n_slots, NG = t.size.n_groups;
    if (!dq->n_queued || !dq->queue_slot || dq->queue_cap < 0 || (NG > 0 && !dq->enforce_after_ns) ||
        (dq->requesting_slot < 0 && NG > 0 && !dq->snapshot_group))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative queue_cap");
    if (dq->requesting_slot < -1 || dq->requesting_slot >= S) return fail(c, GP_ERR_INVALID, who, "requesting_slot outside [-1, n_slots)");
    if (dq->requesting_slot >= 0) {
        if (dq->predicate_group < 0 || dq->predicate_group >= n_sg)
            return fail(c, GP_ERR_INVALID, who, "predicate_group outside the snapshot's groups");
    } else {
        for (int32_t g = 0; g < NG; ++g)
            if (dq->snapshot_group[g] < -1 || dq->snapshot_group[g] >= n_sg)
                return fail(c, GP_ERR_INVALID, who, "a snapshot_group outside [-1, the snapshot's groups)");
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t R = (size_t)S, C = R + 1, G = zones ? (size_t)n_sg : 0;
    Arena ar{t.queue, st};
    const auto keys = ar.take<QueueKey>(R), sorted = ar.take<QueueKey>(R);
    const auto pos = ar.take<int32_t>(R);
    const auto qs = ar.take<int32_t>(C), cnt = ar.take<int32_t>(C), grp = ar.take<int32_t>(C), qidx = ar.take<int32_t>(zones ? C : 0);
    const auto cols = ar.take<long long>(6 * C), cre = ar.take<long long>(C), off = ar.take<long long>(C + 1);
    const auto skip = ar.take<uint8_t>(C);
    const auto sgmap = ar.take<int32_t>(dq->requesting_slot < 0 ? (size_t)NG : 0);
    const auto age = ar.take<long long>((size_t)NG);
    const auto gcount = ar.take<int32_t>(G), gmax = ar.take<int32_t>(G);
    const auto words = ar.take<DqWords>(1);
    ar.reserve();
    ar.zero(gcount); ar.zero(gmax);
    ar.zero(words);
    DqIn in{};
    in.n_rows = S; in.req = dq->requesting_slot; in.scheduler = dq->scheduler; in.pred_group = dq->predicate_group;
    in.sgmap = dq->requesting_slot < 0 ? ar.put(sgmap, dq->snapshot_group) : nullptr;
    in.age = ar.put(age, dq->enforce_after_ns);
    in.now = dq->now_unix_nano;
    GP_TRY(ar.check(c));
    const DtTable T = table_cols(c);
    in.present = T.present; in.exact = T.exact; in.creation = T.creation; in.q = T.q;
    in.sched = T.sched; in.group = T.group; in.count = T.count;
    DqOut o{};
    o.cap = (int32_t)C;
    o.slot = ar.ptr(qs); o.q = ar.ptr(cols); o.count = ar.ptr(cnt); o.group = ar.ptr(grp); o.skip = ar.ptr(skip);
    o.creation = ar.ptr(cre); o.off = ar.ptr(off);
    o.qidx = zones ? ar.ptr(qidx) : nullptr;
    o.gcount = zones ? ar.ptr(gcount) : nullptr; o.gmax = zones ? ar.ptr(gmax) : nullptr;
    DqWords* w = ar.ptr(words);
    if (!t.sort_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<QueueKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(QueueKey))));
        t.sort_attr_set = true;
    }
    if (S > 0) {
        const int rb = (S + kDqThreads - 1) / kDqThreads;
        gp_dq_select<<<rb, kDqThreads, 0, st>>>(in, ar.ptr(keys), w);
        const int32_t* n_sel = &w->selected;
        gp_sort_tiles<QueueKey><<<(S + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(QueueKey), st>>>(S, n_sel, ar.ptr(keys),
                                                                                                                   ar.ptr(sorted));
        gp_rank_by_search<QueueKey><<<rb, kDqThreads, 0, st>>>(S, n_sel, ar.ptr(keys), ar.ptr(sorted), ar.ptr(pos));
        gp_dq_scatter<<<(S + 1 + kDqThreads - 1) / kDqThreads, kDqThreads, 0, st>>>(in, ar.ptr(keys), ar.ptr(pos), w, o);
    }
    gp_dq_finish<<<1, kDqFinishThreads, 0, st>>>(in.req, o, w);
    GP_CUDA(c, cudaGetLastError());
    DqWords hw{};
    ar.get(&hw, words);
    std::vector<int32_t>& hg = c->zone_queue;               // scratch for the counts (fifo_zones_body does not read it)
    hg.assign(2 * G, 0);
    ar.get(hg.data(), gcount);
    ar.get(hg.data() + G, gmax);
    GP_TRY(ar.sync(c));
    *dq->n_queued = hw.n_queued;
    if (dq->n_executors) *dq->n_executors = hw.total;
    if (dq->undefined_ties) *dq->undefined_ties = hw.ties;
    GP_TRY(refuse(c, hw.err, kDqRefusals, who));
    if (hw.n_queued > dq->queue_cap) return fail(c, GP_ERR_CAPACITY, who, "queue_cap too small (*n_queued holds the size needed)");
    if (hw.total > executor_cap)
        return fail(c, GP_ERR_CAPACITY, who, "executor_nodes_cap too small (*n_executors holds the size needed)");
    if (zones) {
        std::vector<ZoneFifoGroup>& zg = c->zone_groups;
        zg.assign(G, ZoneFifoGroup{});
        for (size_t b = 0; b < G; ++b) { zg[b].q_end = hg[b]; zg[b].row_pitch = hg[G + b]; }
    }
    ar.get(dq->queue_slot, ar.ptr(qs), (size_t)hw.n_queued);
    if (dq->exec_out_off) ar.get(dq->exec_out_off, ar.ptr(off), (size_t)hw.n_queued + 1);
    GP_TRY(ar.check(c));
    run->n_queued = hw.n_queued;
    run->total = hw.total;
    run->cols = o;
    return GP_OK;
}

// ---- the marker's stale stage ----

enum : int {
    kDsErrAffinity = 1,         // a stale row's affinity id outside [-1, n_aff)
};

struct DsIn {
    int32_t n_rows, scheduler, n_aff;
    long long timeout, now;
    const uint8_t* present; const uint8_t* exact;
    const long long* creation;
    const long long* q;               // [6][n_rows]
    const int32_t* sched; const int32_t* count; const int32_t* aff;
};

// The stale rows' capacity columns, at their positions in (creation, slot) order; pitch n_rows
struct DsOut {
    int32_t cap;
    int32_t* slot;
    long long* q;                     // [6][cap]
    int32_t* count; int32_t* group;
    uint8_t* outcome;                 // 0, or 2: outside the model (the row is an all-zero placeholder)
};

__global__ void __launch_bounds__(kDqThreads) gp_ds_select(DsIn in, QueueKey* __restrict__ keys, DqWords* __restrict__ w) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    bool sel = false;
    // CreationTimestamp.Add(timeout).Before(now), exactly: creation + timeout < now in 128 bits
    if (r < in.n_rows && in.present[r] && in.sched[r] == in.scheduler)
        sel = (__int128)in.creation[r] + (__int128)in.timeout < (__int128)in.now;
    if (sel && (in.aff[r] < -1 || in.aff[r] >= in.n_aff)) atomicOr(&w->err, kDsErrAffinity);
    const int32_t at = block_compact<kDqThreads>(sel, &w->selected);
    if (sel) {
        QueueKey k; k.sg = 0; k.slot = r; k.creation = in.creation[r];
        keys[at] = k;
    }
}

__global__ void gp_ds_scatter(DsIn in, const QueueKey* __restrict__ keys, const int32_t* __restrict__ pos, const DqWords* __restrict__ w,
                              DsOut o) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w->selected) return;
    const int32_t r = keys[i].slot, p = pos[i];
    const size_t S = (size_t)in.n_rows, C = (size_t)o.cap;
    // what gp_exceeds_cluster_capacity* refuses for a whole call: an inexact row, a negative quantity or count
    bool outside = !in.exact[r] || in.count[r] < 0;
    for (int d = 0; d < 6; ++d) outside |= in.q[(size_t)d * S + r] < 0;
    o.slot[p] = r;
    for (int d = 0; d < 6; ++d) o.q[(size_t)d * C + p] = outside ? 0 : in.q[(size_t)d * S + r];
    o.count[p] = outside ? 0 : in.count[r];
    const int32_t a = in.aff[r];
    o.group[p] = outside || a == -1 ? in.n_aff : a;
    o.outcome[p] = outside ? 2 : 0;
}

gp_status dt_stale_stage(gp_ctx* c, const gp_stale_sweep* sw, int32_t n_aff, const char* who, DtStale* out) {
    auto& t = c->dt;
    const int32_t S = t.size.n_slots;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t R = (size_t)S;
    Arena ar{t.queue, st};
    const auto keys = ar.take<QueueKey>(R), sorted = ar.take<QueueKey>(R);
    const auto pos = ar.take<int32_t>(R), slot = ar.take<int32_t>(R), cnt = ar.take<int32_t>(R), grp = ar.take<int32_t>(R);
    const auto cols = ar.take<long long>(6 * R);
    const auto oc = ar.take<uint8_t>(R);
    const auto words = ar.take<DqWords>(1);
    ar.reserve();
    ar.zero(words);
    GP_TRY(ar.check(c));
    Arena tc{t.cols, st};
    const DtPieces p = take_cols(tc, t.size);
    DsIn in{};
    in.n_rows = S; in.scheduler = sw->scheduler; in.n_aff = n_aff; in.timeout = sw->timeout_ns; in.now = sw->now_unix_nano;
    in.present = tc.ptr(p.present); in.exact = tc.ptr(p.exact); in.creation = tc.ptr(p.creation); in.q = tc.ptr(p.q);
    in.sched = tc.ptr(p.sched); in.count = tc.ptr(p.count); in.aff = tc.ptr(p.aff);
    DsOut o{};
    o.cap = S;
    o.slot = ar.ptr(slot); o.q = ar.ptr(cols); o.count = ar.ptr(cnt); o.group = ar.ptr(grp); o.outcome = ar.ptr(oc);
    DqWords* w = ar.ptr(words);
    if (!t.sort_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<QueueKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(QueueKey))));
        t.sort_attr_set = true;
    }
    if (S > 0) {
        const int rb = (S + kDqThreads - 1) / kDqThreads;
        gp_ds_select<<<rb, kDqThreads, 0, st>>>(in, ar.ptr(keys), w);
        const int32_t* n_sel = &w->selected;
        gp_sort_tiles<QueueKey><<<(S + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(QueueKey), st>>>(S, n_sel, ar.ptr(keys),
                                                                                                                   ar.ptr(sorted));
        gp_rank_by_search<QueueKey><<<rb, kDqThreads, 0, st>>>(S, n_sel, ar.ptr(keys), ar.ptr(sorted), ar.ptr(pos));
        gp_ds_scatter<<<rb, kDqThreads, 0, st>>>(in, ar.ptr(keys), ar.ptr(pos), w, o);
    }
    GP_CUDA(c, cudaGetLastError());
    DqWords hw{};
    ar.get(&hw, words);
    GP_TRY(ar.sync(c));
    static const Refusal refusals[] = {{kDsErrAffinity, GP_ERR_INVALID, "a stale driver's affinity id outside [-1, n_aff)"}};
    GP_TRY(refuse(c, hw.err, refusals, who));
    *sw->n_stale = hw.selected;
    if (hw.selected > sw->cap) return fail(c, GP_ERR_CAPACITY, who, "cap too small (*n_stale holds the size needed)");
    // completed by the capacity call's synchronise
    const size_t n = (size_t)hw.selected;
    ar.get(sw->stale_slot, ar.ptr(slot), n);
    ar.get(sw->outcome, ar.ptr(oc), n);
    GP_TRY(ar.check(c));
    *out = DtStale{};
    out->n = hw.selected;
    for (int d = 0; d < 6; ++d) out->q[d] = (const int64_t*)o.q + (size_t)d * R;
    out->count = o.count;
    out->group = o.group;
    return GP_OK;
}

extern "C" {

gp_status gp_driver_table_reset(gp_ctx* c, const gp_driver_table_size* z) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_driver_table_reset";
    if (!z || z->n_slots < 0 || z->n_groups < 0 || z->n_schedulers < 0) return fail(c, GP_ERR_INVALID, who, "NULL size or a negative capacity");
    return c->dt.reset(c, *z, [&](Arena& a) {
        const DtPieces p = take_cols(a, *z);
        a.reserve();
        a.fill(p.present, p.stamp, 0);
        return GP_OK;
    });
}

gp_status gp_driver_table_update(gp_ctx* c, const gp_driver_delta* d) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_driver_table_update";
    auto& t = c->dt;
    GP_TRY(require(c, t.need(), who));
    if (!d || d->n_write < 0 ||
        (d->n_write > 0 && (!d->slot || !d->present || !d->creation || !d->scheduler || !d->group || !d->drv_cpu_milli ||
                            !d->drv_mem_bytes || !d->exe_cpu_milli || !d->exe_mem_bytes || !d->min_executor_count || !d->exact)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative count");
    if (d->n_write > t.size.n_slots) return fail(c, GP_ERR_INVALID, who, "more writes than slots: a slot given twice or out of range");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t W = (size_t)d->n_write;
    Arena ar{c->callbuf, st};
    const auto slot = ar.take<int32_t>(W), sched = ar.take<int32_t>(W), grp = ar.take<int32_t>(W), cnt = ar.take<int32_t>(W);
    const auto aff = ar.take<int32_t>(W);
    const auto on = ar.take<uint8_t>(W), ex = ar.take<uint8_t>(W);
    const auto cre = ar.take<long long>(W), q = ar.take<long long>(6 * W);
    const auto word = ar.take<int>(1);
    ar.reserve();
    ar.zero(word);
    DtDelta D{};
    D.n = d->n_write; D.n_rows = t.size.n_slots; D.n_groups = t.size.n_groups; D.n_sched = t.size.n_schedulers;
    D.slot = ar.put(slot, d->slot);
    D.present = ar.put(on, d->present);
    D.creation = ar.put(cre, d->creation);
    D.sched = ar.put(sched, d->scheduler);
    D.group = ar.put(grp, d->group);
    const int64_t* hq[6] = {d->drv_cpu_milli, d->drv_mem_bytes, d->drv_gpu, d->exe_cpu_milli, d->exe_mem_bytes, d->exe_gpu};
    for (int k = 0; k < 6; ++k) D.q[k] = ar.put(q.part((size_t)k * W, W), hq[k]);
    D.count = ar.put(cnt, d->min_executor_count);
    D.exact = ar.put(ex, d->exact);
    const int32_t* d_aff = ar.put(aff, d->affinity);
    GP_TRY(ar.check(c));
    Arena tc{t.cols, st};
    const DtPieces p = take_cols(tc, t.size);
    GP_TRY(t.begin(c, tc, p.stamp, p.stamp));
    int* w = ar.ptr(word);
    if (W > 0) {
        const int T = 256;
        const unsigned wb = (unsigned)((W + T - 1) / T);
        gp_dt_check<<<wb, T, 0, st>>>(D, tc.ptr(p.stamp), t.seq, w);
        gp_dt_apply<<<wb, T, 0, st>>>(D, table_cols(c), w);
        gp_dt_apply_aff<<<wb, T, 0, st>>>(D.n, D.slot, D.present, d_aff, table_aff(c), w);
    }
    int hw = 0;
    return t.commit(c, ar, word, &hw, kDtRefusals, who);
}

gp_status gp_pack_fifo_driver_table(gp_ctx* c, const gp_driver_queue* dq, gp_algo algo, gp_mode mode, gp_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_pack_fifo_driver_table";
    // gp_pack_batch's checks for the FIFO modes
    GP_TRY(require(c, c->held.snapshot(), who));
    if (!dq || !out) return fail(c, GP_ERR_INVALID, who, "NULL queue/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_DISTRIBUTE_EVENLY) return fail(c, GP_ERR_INVALID, who, "algo must be tightly-pack or distribute-evenly");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT) return fail(c, GP_ERR_INVALID, who, "mode must be one of the FIFO modes");
    if (!out->driver_node) return fail(c, GP_ERR_INVALID, who, "missing result arrays");
    QueueRun run{};
    GP_TRY(queue_stage(c, dq, c->n_groups, false, out->executor_nodes_cap, who, &run));
    const int32_t q = run.n_queued;
    if (q == 0) return GP_OK;
    if (run.total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, who, "executor_nodes is NULL");
    cudaStream_t st = c->stream;
    GP_CUDA(c, c->r_driver.reserve(sizeof(int32_t) * (size_t)q));
    GP_CUDA(c, c->r_exec.reserve(sizeof(int32_t) * (size_t)(run.total + 1)));
    int2* scratch = nullptr;
    GP_TRY(pack_begin(c, q, algo, mode, out->executor_nodes_cap, false, &scratch, st));
    const DqOut& o = run.cols;
    const size_t C = (size_t)o.cap;
    DevApps dv{};
    for (int k = 0; k < 6; ++k) dv.cols.q[k] = o.q + (size_t)k * C;
    dv.cols.count = o.count; dv.cols.group = o.group; dv.cols.off = (const int64_t*)o.off; dv.cols.bits = 64; dv.cols.mem_shift = 0;
    dv.skip = o.skip; dv.n = q;
    DevResults dr{c->r_driver.as<int32_t>(), c->r_exec.p, out->executor_nodes_cap, 32};
    GP_TRY(pack_device_range(c, dv, 0, q, 0, algo, mode, dr, scratch, st, 0));
    c->ev_chunks = 1;
    Arena ar{c->r_driver, st};
    ar.get(out->driver_node, c->r_driver.as<int32_t>(), (size_t)q);
    ar.get(out->executor_nodes, c->r_exec.as<int32_t>(), (size_t)run.total);
    GP_TRY(ar.sync(c));
    return host_error(c);
}

gp_status gp_pack_fifo_zones_groups_driver_table(gp_ctx* c, const gp_driver_queue* dq, gp_binpacker packer, gp_mode mode,
                                                 const gp_instance_groups* groups, gp_zone_results* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_pack_fifo_zones_groups_driver_table";
    GP_TRY(require(c, c->held.snapshot(), who));
    int kind;
    GP_TRY(zone_fifo_kind(c, packer, mode, who, &kind));
    if (groups) return fail(c, GP_ERR_INVALID, who, "groups must be NULL: the layout gp_prepare_cluster_zones_groups left");
    if (!dq || !out) return fail(c, GP_ERR_INVALID, who, "NULL queue/results");
    gp_instance_groups held{};
    GP_TRY(held_groups_layout(c, kind, who, &held));
    if (!out->zone || !out->driver_node) return fail(c, GP_ERR_INVALID, who, "missing result arrays");
    QueueRun run{};
    GP_TRY(queue_stage(c, dq, held.n_instance_groups, true, out->executor_nodes_cap, who, &run));
    if (run.n_queued == 0) return GP_OK;
    const DqOut& o = run.cols;
    ZoneFifoApps src{};
    for (int k = 0; k < 6; ++k) src.q[k] = (const int64_t*)o.q + (size_t)k * (size_t)o.cap;
    src.count = o.count; src.off = (const int64_t*)o.off; src.skip = o.skip; src.queue = o.qidx;
    return fifo_zones_body(c, run.n_queued, run.total, src, kind, mode, held, kind == kZoneAzAware, out, who);
}

}  // extern "C"
