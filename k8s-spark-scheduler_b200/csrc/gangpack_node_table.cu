// gangpack_node_table.cu -- the resident node table: gp_node_table_reset and gp_node_table_update, and the gather of the
// *_node_table entries (gangpack_cluster.cu), which read it in place.
//
// An update runs
//   gp_nt_keys      thread per row: the row's NameKey (name_key, id) as the table holds it, absent rows last
//   gp_nt_check     thread per row write: node id range, duplicates (per-row stamps, stamped_twice), |alloc| < 2^61 and
//                   name_key < 2^63 - 1 on present rows; then the write's key replaces its row's key in the scratch, so the
//                   scratch holds the table as it will be after the delta
//   gp_sort_tiles / gp_rank_by_search <NameKey>   pos[row] = the row's rank among all rows by (name_key, id)
//   gp_nt_scatter + gp_nt_dups   the keys in rank order; two adjacent present keys that are equal refuse the delta
//   gp_nt_apply     the row writes and name_rank[row] = pos[row] (-1 absent); nothing when the error word is set
//   gp_nt_creation  the rows' creation times, under the same condition
// within the update protocol of gangpack_resident.cuh, so a refused delta leaves the table as it was.
//
// The gather (gp_nt_gather, thread per listed node) writes exactly the columns a *_resident entry would upload: allocatable,
// name_rank, unschedulable and ready from the node table, and zone, instance group and the two label ranks from the label
// table's row of the same id, read through AffLabelsResident's row range and aff_find.  For the failover reconciler it also
// writes creation, and reads the instance group under the reconciler's rule (a missing label is the group of "").
#include "gangpack_ctx.cuh"
#include "gangpack_labels.cuh"
#include "gangpack_tilesort.cuh"

#include <algorithm>
#include <vector>

namespace gp {

// the rank key of a row: (name_key, id) in 12 bytes (a tile of 4 096 is 48 KB, the default dynamic shared-memory limit)
struct NameKey {
    int32_t hi;           // name_key's high half (signed)
    uint32_t lo;          // its low half
    int32_t id;
};
__device__ __forceinline__ bool key_less(const NameKey& a, const NameKey& b) {
    return a.hi != b.hi ? a.hi < b.hi : (a.lo != b.lo ? a.lo < b.lo : a.id < b.id);
}
__device__ __forceinline__ NameKey key_max(const NameKey*) { NameKey k; k.hi = 0x7fffffff; k.lo = 0xffffffffu; k.id = 0x7fffffff; return k; }

}  // namespace gp

static constexpr long long kAbsentKey = 0x7fffffffffffffffLL;      // the key of an absent row: after every present one

__device__ __forceinline__ NameKey name_key_of(long long key, int32_t id) {
    NameKey k; k.hi = (int32_t)(key >> 32); k.lo = (uint32_t)key; k.id = id;
    return k;
}
__device__ __forceinline__ long long key_value(const NameKey& k) { return (long long)(((unsigned long long)(uint32_t)k.hi << 32) | k.lo); }

enum : int {
    kNtErrRange = 1,            // a node id out of range
    kNtErrDuplicate = 2,        // a node id given twice
    kNtErrKey = 4,              // two present rows with one name_key, or a present name_key of 2^63 - 1
    kNtErrInput = 8,            // |alloc| >= 2^61 on a present row
};

static const Refusal kNtRefusals[] = {
    {kNtErrRange, GP_ERR_INVALID, "a node id out of range"},
    {kNtErrDuplicate, GP_ERR_INVALID, "a node id given twice"},
    {kNtErrKey, GP_ERR_INVALID, "two present rows with the same name_key, or a name_key of 2^63 - 1"},
    {kNtErrInput, GP_ERR_UNREPRESENTABLE, "|alloc| >= 2^61 on a present row"},
};

struct NtPieces {
    Piece<uint8_t> present, unsched, ready;
    Piece<long long> alloc, key, creation;
    Piece<int32_t> rank;
    Piece<uint32_t> stamp;
};

// The layout of the table's column block (all 0 after a reset: no row present; rank is written by every update)
static NtPieces take_cols(Arena& a, const gp_node_table_size& z) {
    const size_t R = (size_t)z.n_node_ids;
    NtPieces p;
    p.present = a.take<uint8_t>(R);
    p.unsched = a.take<uint8_t>(R);
    p.ready = a.take<uint8_t>(R);
    p.alloc = a.take<long long>(3 * R);
    p.key = a.take<long long>(R);
    p.creation = a.take<long long>(R);
    p.rank = a.take<int32_t>(R);
    p.stamp = a.take<uint32_t>(R);
    return p;
}

// One update, staged on the device
struct NtDelta {
    int32_t n, n_rows;
    const int32_t* id;
    const uint8_t* present;
    const long long* alloc[3];        // alloc[2] NULL: 0
    const uint8_t* unsched;
    const uint8_t* ready;
    const long long* key;
    const long long* creation;        // NULL: 0
};

struct NtTable {
    uint8_t* present; uint8_t* unsched; uint8_t* ready;
    long long* alloc;                 // [3][n_rows]
    long long* key;
    int32_t* rank;
};

__global__ void gp_nt_keys(int32_t R, const uint8_t* __restrict__ present, const long long* __restrict__ key, NameKey* __restrict__ keys) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R) keys[r] = name_key_of(present[r] ? key[r] : kAbsentKey, r);
}

__global__ void gp_nt_check(NtDelta D, uint32_t* __restrict__ stamp, uint32_t seq, NameKey* __restrict__ keys, int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.n) return;
    const int32_t r = D.id[i];
    if (r < 0 || r >= D.n_rows) { atomicOr(err, kNtErrRange); return; }
    int bad = stamped_twice(stamp + r, seq) ? kNtErrDuplicate : 0;
    const bool on = D.present[i] != 0;
    if (on) {
        for (int d = 0; d < 3; ++d)
            if (D.alloc[d] && (D.alloc[d][i] <= -kMaxQuantity || D.alloc[d][i] >= kMaxQuantity)) bad |= kNtErrInput;
        if (D.key[i] == kAbsentKey) bad |= kNtErrKey;
    }
    keys[r] = name_key_of(on ? D.key[i] : kAbsentKey, r);
    if (bad) atomicOr(err, bad);
}

// skey[pos[r]] = the key value of row r: the keys in rank order
__global__ void gp_nt_scatter(int32_t R, const NameKey* __restrict__ keys, const int32_t* __restrict__ pos, long long* __restrict__ skey) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R) skey[pos[r]] = key_value(keys[r]);
}

__global__ void gp_nt_dups(int32_t R, const long long* __restrict__ skey, int* __restrict__ err) {
    const int32_t p = blockIdx.x * blockDim.x + threadIdx.x + 1;
    if (p < R && skey[p] != kAbsentKey && skey[p] == skey[p - 1]) atomicOr(err, kNtErrKey);
}

__global__ void gp_nt_apply(NtDelta D, NtTable T, const NameKey* __restrict__ keys, const int32_t* __restrict__ pos,
                            const int* __restrict__ err) {
    if (*(volatile const int*)err) return;
    const long long total = (long long)D.n + D.n_rows;
    const size_t R = (size_t)D.n_rows;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < D.n) {
            const int32_t r = D.id[i];
            const bool on = D.present[i] != 0;
            T.present[r] = on ? 1 : 0;
            for (int d = 0; d < 3; ++d) T.alloc[(size_t)d * R + r] = on && D.alloc[d] ? D.alloc[d][i] : 0;
            T.unsched[r] = on && D.unsched[i] ? 1 : 0;
            T.ready[r] = on && D.ready[i] ? 1 : 0;
            T.key[r] = on ? D.key[i] : 0;
        } else {
            const int32_t r = (int32_t)(i - D.n);
            T.rank[r] = key_value(keys[r]) == kAbsentKey ? -1 : pos[r];
        }
    }
}

// creation[row] of every write (0 for a deleted row), when the delta was accepted.  A kernel of its own, so that gp_nt_apply
// is compiled as it was before the table kept creation times.
__global__ void gp_nt_creation(NtDelta D, long long* __restrict__ creation, const int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.n || *(volatile const int*)err) return;
    creation[D.id[i]] = D.present[i] && D.creation ? D.creation[i] : 0;
}

// ---- the gather of the *_node_table entries ----

enum : int {
    kNtgErrId = 1,              // a node-table id out of range, absent or given twice
    kNtgErrZone = 2,            // a zone value not listed, or a node without the zone label and zone_missing = -1
    kNtgErrGroup = 4,           // the reconciler's rule: an instance-group value not listed
    kNtgErrGroupMissing = 8,    // the reconciler's rule: a node without the instance-group label and instance_group_missing = -1
};

static const Refusal kNtgRefusals[] = {
    {kNtgErrId, GP_ERR_INVALID, "a node-table id out of range, absent or given twice"},
    {kNtgErrZone, GP_ERR_INVALID, "a zone label value not in zone_value, or a node without the zone label (zone_missing = -1)"},
    {kNtgErrGroup, GP_ERR_INVALID, "an instance-group label value not in instance_group_value"},
    {kNtgErrGroupMissing, GP_ERR_INVALID, "a node without the instance-group label (instance_group_missing = -1)"},
};

// A label key and the value ids it maps: map [n] sorted by value, .y = the dense id or rank.  key -1: not read.
struct NtLabelMap {
    int32_t key, n;
    const int2* map;
};

struct NtGatherIn {
    int32_t n, n_rows;
    const int32_t* id;                // [n] node-table ids
    AffLabelsResident L;              // node_id = id
    const uint8_t* present; const uint8_t* unsched; const uint8_t* ready;
    const long long* alloc;           // [3][n_rows]
    const int32_t* rank;
    const long long* creation;        // [n_rows]
    NtLabelMap zone, ig, lr[2];
    int32_t zone_missing;
    int32_t ig_missing;               // the reconciler's rule (strict_ig): the group of a node without the label, -1 refused
    bool strict_ig;
    int32_t* dir;                     // [n_rows] -1: no listed node has the id yet
    long long* alloc_out;             // [3][n]
    int32_t* rank_out; uint8_t* unsched_out; uint8_t* ready_out;
    int32_t* zone_out; int32_t* ig_out; int32_t* lr_out[2];
    long long* creation_out;          // [n] or NULL: not asked for
    int* err;
};

// the dense id of value v in m, -1 when it is not listed
__device__ __forceinline__ int32_t nt_lookup(const NtLabelMap& m, int32_t v) {
    int32_t lo = 0, hi = m.n;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        const int2 e = m.map[mid];
        if (e.x == v) return e.y;
        if (e.x < v) lo = mid + 1; else hi = mid;
    }
    return -1;
}

// the value id of label `key` of listed node i, -1 when the node does not have it
__device__ __forceinline__ int32_t nt_label(const AffLabelsResident& L, int32_t i, int32_t key) {
    long long lo, hi;
    L.range(i, lo, hi);
    const long long e = aff_find(L.key, lo, hi, key);
    return e < 0 ? -1 : L.val[e];
}

__global__ void gp_nt_gather(NtGatherIn G) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G.n) return;
    const int32_t r = G.id[i];
    int bad = 0;
    const bool present = r >= 0 && r < G.n_rows && G.present[r];
    // the first listed entry of a present row owns it; any other entry is refused
    const bool ok = present && atomicCAS(G.dir + r, -1, i) == -1;
    if (!ok) bad |= kNtgErrId;
    const size_t N = (size_t)G.n, R = (size_t)G.n_rows;
    for (int d = 0; d < 3; ++d) G.alloc_out[(size_t)d * N + i] = ok ? G.alloc[(size_t)d * R + r] : 0;
    // The stages after the gather run before its refusal is read, and their sort needs name ranks that are unique (a rank
    // given twice leaves a position of the order unwritten).  The owners' table ranks are distinct and >= 0; every refused
    // entry takes -1 - i, distinct from them and from each other.
    G.rank_out[i] = ok ? G.rank[r] : -1 - i;
    G.unsched_out[i] = ok ? G.unsched[r] : 0;
    G.ready_out[i] = ok ? G.ready[r] : 0;
    if (G.zone.key >= 0) {
        const int32_t v = nt_label(G.L, i, G.zone.key);
        int32_t z = v < 0 ? G.zone_missing : nt_lookup(G.zone, v);
        if (z < 0) { bad |= kNtgErrZone; z = 0; }
        G.zone_out[i] = z;
    }
    if (G.creation_out) G.creation_out[i] = ok ? G.creation[r] : 0;
    if (G.strict_ig) {
        // every node in [0, n_groups): a refused one takes 0, so that the reconciler's stages index in range
        int32_t g = 0;
        if (G.ig.key >= 0) {
            const int32_t v = nt_label(G.L, i, G.ig.key);
            g = v < 0 ? G.ig_missing : nt_lookup(G.ig, v);
            if (g < 0) { bad |= v < 0 ? kNtgErrGroupMissing : kNtgErrGroup; g = 0; }
        }
        G.ig_out[i] = g;
    } else if (G.ig.key >= 0) {
        const int32_t v = nt_label(G.L, i, G.ig.key);
        G.ig_out[i] = v < 0 ? -1 : nt_lookup(G.ig, v);
    }
    for (int k = 0; k < 2; ++k)
        if (G.lr[k].key >= 0) {
            const int32_t v = nt_label(G.L, i, G.lr[k].key);
            G.lr_out[k][i] = v < 0 ? -1 : nt_lookup(G.lr[k], v);
        }
    if (bad) atomicOr(G.err, bad);
}

// (value, dense id) of list[n] sorted by value; a value listed twice is refused (distinct) or keeps its last index (ranks)
static bool label_map(const int32_t* list, int32_t n, bool distinct, std::vector<int2>& out) {
    out.clear();
    for (int32_t k = 0; k < n; ++k) out.push_back(make_int2(list[k], k));
    std::sort(out.begin(), out.end(), [](int2 a, int2 b) { return a.x != b.x ? a.x < b.x : a.y < b.y; });
    std::vector<int2> kept;
    for (size_t k = 0; k < out.size(); ++k) {
        if (k + 1 < out.size() && out[k + 1].x == out[k].x) {
            if (distinct) return false;
            continue;                                   // the later index wins, as valueRanks[value] = i does
        }
        kept.push_back(out[k]);
    }
    out.swap(kept);
    return true;
}

gp_status nt_gather(gp_ctx* c, const gp_node_table_nodes* nd, const int32_t* ig_host, int32_t n_ig, bool with_ig, const char* who,
                    NtGathered* g, const NtReconcile* recon, bool reservations) {
    auto& t = c->nt;
    GP_TRY(require(c, t.need(), c->lt.need(), who));
    if (!nd || nd->n_nodes < 0 || nd->n_zones < 1 ||
        (nd->n_nodes > 0 && (!nd->node_table_id || (reservations && !nd->reservation_id) || !nd->overhead_node_id)) ||
        (nd->zone_key >= 0 && !nd->zone_value) || (with_ig && !ig_host && nd->instance_group_key >= 0 && n_ig > 0 && !nd->instance_group_value) ||
        (nd->driver_rank_key >= 0 && (nd->n_driver_rank_values < 0 || (nd->n_driver_rank_values > 0 && !nd->driver_rank_value))) ||
        (nd->executor_rank_key >= 0 && (nd->n_executor_rank_values < 0 || (nd->n_executor_rank_values > 0 && !nd->executor_rank_value))))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or bad sizes");
    if (nd->zone_missing < -1 || nd->zone_missing >= nd->n_zones) return fail(c, GP_ERR_INVALID, who, "zone_missing outside [-1, n_zones)");
    if (recon && (recon->missing < -1 || recon->missing >= std::max(n_ig, 0)))
        return fail(c, GP_ERR_INVALID, who, "instance_group_missing outside [-1, n_groups)");
    const bool label_ig = with_ig && !ig_host && nd->instance_group_key >= 0;
    std::vector<int2> maps[4];
    if (nd->zone_key >= 0 && !label_map(nd->zone_value, nd->n_zones, true, maps[0]))
        return fail(c, GP_ERR_INVALID, who, "a value listed twice in zone_value");
    if (label_ig && !label_map(nd->instance_group_value, std::max(n_ig, 0), true, maps[1]))
        return fail(c, GP_ERR_INVALID, who, "a value listed twice in instance_group_value");
    if (nd->driver_rank_key >= 0) label_map(nd->driver_rank_value, nd->n_driver_rank_values, false, maps[2]);
    if (nd->executor_rank_key >= 0) label_map(nd->executor_rank_value, nd->n_executor_rank_values, false, maps[3]);
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const int32_t n = nd->n_nodes;
    const size_t N = (size_t)n, R = (size_t)t.size.n_node_ids;
    Arena ar{t.gather, st};
    const auto id = ar.take<int32_t>(N);
    const auto alloc = ar.take<long long>(3 * N);
    const auto rank = ar.take<int32_t>(N), zone = ar.take<int32_t>(N), ig = ar.take<int32_t>(N), lrd = ar.take<int32_t>(N),
               lre = ar.take<int32_t>(N);
    const auto fu = ar.take<uint8_t>(N), fr = ar.take<uint8_t>(N);
    const auto cre = ar.take<long long>(recon ? N : 0);
    const auto dir = ar.take<int32_t>(R);
    Piece<int2> mp[4];
    for (int k = 0; k < 4; ++k) mp[k] = ar.take<int2>(maps[k].size());
    const auto err = ar.take<int>(1);
    ar.reserve();
    NtGatherIn G{};
    G.n = n; G.n_rows = t.size.n_node_ids;
    G.id = ar.put(id, nd->node_table_id);
    const LtCols lc = lt_cols(c);
    G.L.n = n; G.L.n_rows = c->lt.size.n_node_ids; G.L.stride = c->lt.size.max_labels; G.L.node_id = G.id;
    G.L.count = lc.count; G.L.key = lc.key; G.L.val = lc.val; G.L.val_int_ok = lc.vok; G.L.val_int = lc.vint;
    Arena tc{t.cols, st};
    const NtPieces p = take_cols(tc, t.size);
    G.present = tc.ptr(p.present); G.unsched = tc.ptr(p.unsched); G.ready = tc.ptr(p.ready);
    G.alloc = tc.ptr(p.alloc); G.rank = tc.ptr(p.rank); G.creation = tc.ptr(p.creation);
    const int32_t keys[4] = {nd->zone_key, label_ig ? nd->instance_group_key : -1, nd->driver_rank_key, nd->executor_rank_key};
    NtLabelMap* lm[4] = {&G.zone, &G.ig, &G.lr[0], &G.lr[1]};
    for (int k = 0; k < 4; ++k) *lm[k] = NtLabelMap{keys[k] >= 0 ? keys[k] : -1, (int32_t)maps[k].size(), ar.put(mp[k], maps[k].data())};
    G.zone_missing = nd->zone_missing;
    G.strict_ig = recon != nullptr;
    G.ig_missing = recon ? recon->missing : -1;
    G.creation_out = recon ? ar.ptr(cre) : nullptr;
    G.dir = ar.fill(dir, 0xff);
    G.alloc_out = ar.ptr(alloc); G.rank_out = ar.ptr(rank); G.unsched_out = ar.ptr(fu); G.ready_out = ar.ptr(fr);
    G.zone_out = ar.ptr(zone); G.ig_out = ar.ptr(ig); G.lr_out[0] = ar.ptr(lrd); G.lr_out[1] = ar.ptr(lre);
    G.err = ar.zero(err);
    if (ig_host) ar.put(ig, ig_host);
    GP_TRY(ar.check(c));
    const int T = 256;
    if (n > 0) gp_nt_gather<<<(n + T - 1) / T, T, 0, st>>>(G);
    GP_CUDA(c, cudaGetLastError());

    gp_resident_usage& u = g->usage;
    u = gp_resident_usage{};
    u.n_nodes = n;
    u.node_id = nd->reservation_id;
    u.alloc_cpu_milli = (const int64_t*)G.alloc_out;
    u.alloc_mem_bytes = (const int64_t*)G.alloc_out + N;
    u.alloc_gpu = (const int64_t*)G.alloc_out + 2 * N;
    u.overhead_node_id = nd->overhead_node_id;
    gp_sort_input& s = g->sort;
    s = gp_sort_input{};
    s.n_nodes = n;
    s.n_zones = nd->n_zones;
    s.zone_id = nd->zone_key >= 0 ? G.zone_out : nullptr;
    s.name_rank = G.rank_out;
    s.is_driver_candidate = nd->is_driver_candidate;
    s.unschedulable = G.unsched_out;
    s.ready = G.ready_out;
    s.driver_label_rank = nd->driver_rank_key >= 0 ? G.lr_out[0] : nullptr;
    s.executor_label_rank = nd->executor_rank_key >= 0 ? G.lr_out[1] : nullptr;
    s.undefined_ties = nd->undefined_ties;
    g->ig = ig_host || label_ig || recon ? G.ig_out : nullptr;
    g->creation = G.creation_out;
    g->err = G.err;
    return GP_OK;
}

gp_status nt_refusal(gp_ctx* c, int word, const char* who) { return refuse(c, word, kNtgRefusals, who); }

gp_status nt_outputs(gp_ctx* c, const gp_node_table_nodes* nd, const NtGathered& g) {
    const size_t N = (size_t)nd->n_nodes;
    if (nd->zone_id_out && !g.sort.zone_id) std::fill(nd->zone_id_out, nd->zone_id_out + N, 0);
    if (nd->instance_group_out && !g.ig) std::fill(nd->instance_group_out, nd->instance_group_out + N, 0);
    Arena ar{c->nt.gather, c->stream};
    if (g.sort.zone_id) ar.get(nd->zone_id_out, g.sort.zone_id, N);
    if (g.ig) ar.get(nd->instance_group_out, g.ig, N);
    if ((nd->zone_id_out && g.sort.zone_id) || (nd->instance_group_out && g.ig)) GP_TRY(ar.sync(c));
    return GP_OK;
}

extern "C" {

gp_status gp_node_table_reset(gp_ctx* c, const gp_node_table_size* z) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_node_table_reset";
    if (!z || z->n_node_ids < 0) return fail(c, GP_ERR_INVALID, who, "NULL size or a negative capacity");
    return c->nt.reset(c, *z, [&](Arena& a) {
        const NtPieces p = take_cols(a, *z);
        a.reserve();
        a.fill(p.present, p.stamp, 0);
        return GP_OK;
    });
}

gp_status gp_node_table_update(gp_ctx* c, const gp_node_delta* d) {
    if (!enter(c)) return GP_ERR_INVALID;
    static const char* who = "gp_node_table_update";
    auto& t = c->nt;
    GP_TRY(require(c, t.need(), who));
    if (!d || d->n_write < 0 ||
        (d->n_write > 0 && (!d->node_id || !d->present || !d->alloc_cpu_milli || !d->alloc_mem_bytes || !d->unschedulable ||
                            !d->ready || !d->name_key)))
        return fail(c, GP_ERR_INVALID, who, "missing arrays or a negative count");
    if (d->n_write > t.size.n_node_ids) return fail(c, GP_ERR_INVALID, who, "more writes than rows: a node id given twice or out of range");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t W = (size_t)d->n_write, R = (size_t)t.size.n_node_ids;
    const int32_t n_rows = t.size.n_node_ids;
    Arena ar{c->callbuf, st};
    const auto id = ar.take<int32_t>(W);
    const auto on = ar.take<uint8_t>(W), fu = ar.take<uint8_t>(W), fr = ar.take<uint8_t>(W);
    const auto al = ar.take<long long>(3 * W), key = ar.take<long long>(W), cre = ar.take<long long>(W);
    const auto keys = ar.take<NameKey>(R), sorted = ar.take<NameKey>(R);
    const auto pos = ar.take<int32_t>(R);
    const auto skey = ar.take<long long>(R);
    const auto word = ar.take<int>(1);
    ar.reserve();
    ar.zero(word);
    NtDelta D{};
    D.n = d->n_write; D.n_rows = n_rows;
    D.id = ar.put(id, d->node_id);
    D.present = ar.put(on, d->present);
    D.alloc[0] = ar.put(al.part(0, W), d->alloc_cpu_milli);
    D.alloc[1] = ar.put(al.part(W, W), d->alloc_mem_bytes);
    D.alloc[2] = ar.put(al.part(2 * W, W), d->alloc_gpu);
    D.unsched = ar.put(fu, d->unschedulable);
    D.ready = ar.put(fr, d->ready);
    D.key = ar.put(key, d->name_key);
    D.creation = ar.put(cre, d->creation);
    GP_TRY(ar.check(c));
    Arena tc{t.cols, st};
    const NtPieces p = take_cols(tc, t.size);
    GP_TRY(t.begin(c, tc, p.stamp, p.stamp));
    int* w = ar.ptr(word);
    const int T = 256;
    if (R > 0) {
        const int rb = (int)((R + T - 1) / T);
        gp_nt_keys<<<rb, T, 0, st>>>(n_rows, tc.ptr(p.present), tc.ptr(p.key), ar.ptr(keys));
        if (W > 0) gp_nt_check<<<(unsigned)((W + T - 1) / T), T, 0, st>>>(D, tc.ptr(p.stamp), t.seq, ar.ptr(keys), w);
        gp_sort_tiles<NameKey><<<(n_rows + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(NameKey), st>>>(n_rows, nullptr, ar.ptr(keys),
                                                                                                                   ar.ptr(sorted));
        gp_rank_by_search<NameKey><<<rb, T, 0, st>>>(n_rows, nullptr, ar.ptr(keys), ar.ptr(sorted), ar.ptr(pos));
        gp_nt_scatter<<<rb, T, 0, st>>>(n_rows, ar.ptr(keys), ar.ptr(pos), ar.ptr(skey));
        gp_nt_dups<<<rb, T, 0, st>>>(n_rows, ar.ptr(skey), w);
        const NtTable tab{tc.ptr(p.present), tc.ptr(p.unsched), tc.ptr(p.ready), tc.ptr(p.alloc), tc.ptr(p.key), tc.ptr(p.rank)};
        const long long items = (long long)W + (long long)R;
        gp_nt_apply<<<update_grid(items, T, c->sm_count), T, 0, st>>>(D, tab, ar.ptr(keys), ar.ptr(pos), w);
        if (W > 0) gp_nt_creation<<<(unsigned)((W + T - 1) / T), T, 0, st>>>(D, tc.ptr(p.creation), w);
    }
    int hw = 0;
    return t.commit(c, ar, word, &hw, kNtRefusals, who);
}

}  // extern "C"
