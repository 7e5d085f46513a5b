// gangpack_placement.cu -- the driver Predicate's placement metrics: gp_placement_metrics (host arrays) and
// gp_placement_metrics_device (device arrays, asynchronous), one set of kernels (gangpack_placement.cuh).
#include "gangpack_ctx.cuh"
#include "gangpack_placement.cuh"

#include <algorithm>
#include <vector>

static constexpr size_t kPmGlobalScratch = (size_t)256 << 20;   // bytes of global-scratch slices one launch may take

// The placement kernels' status word (kPmErr* bits)
static const Refusal kPmRefusals[] = {
    {kPmErrCount, GP_ERR_INVALID, "negative exe_count"},
    {kPmErrGroup, GP_ERR_INVALID, "instance_group outside [-1, n_instance_groups) or apps->group outside [0, n_instance_groups)"},
    {kPmErrNode, GP_ERR_INVALID, "a placed row's driver or executor node outside [0, n_nodes)"},
    {kPmErrZone, GP_ERR_INVALID, "metric_zone outside [0, n_metric_zones)"},
    {kPmErrUnrepresentable, GP_ERR_UNREPRESENTABLE, "exe_count above 2^24"},
    {kPmErrCapacity, GP_ERR_CAPACITY, "a placed row's ExecutorNodes outside executor_nodes_cap"},
};

// Launch shapes: a slice per team, in dynamic shared memory when it fits, in global scratch otherwise
struct PmPlan {
    int32_t bitmap_words;
    long long slice_words;
    size_t slice_bytes;
    int warp_block, warp_grid, cta_grid;
    size_t warp_smem, cta_smem;
    bool warp_global, cta_global;
    size_t global_slices;            // slices of global scratch (the larger of the two kernels' needs)
};

static gp_status pm_plan(gp_ctx* c, int32_t N, int32_t Z, int32_t Q, PmPlan& p) {
    if (!c->pm_smem_limit) {
        int optin = 0;
        GP_CUDA(c, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
        const int limit = optin - 1024;                          // room for the kernels' static shared memory
        GP_CUDA(c, cudaFuncSetAttribute(gp_placement_rows<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit));
        GP_CUDA(c, cudaFuncSetAttribute(gp_placement_rows<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit));
        c->pm_smem_limit = limit;
    }
    const size_t limit = (size_t)c->pm_smem_limit, sm = (size_t)c->sm_count;
    p.bitmap_words = (int32_t)(((int64_t)N + 31) / 32);
    p.slice_words = (long long)p.bitmap_words + Z;
    p.slice_bytes = sizeof(uint32_t) * (size_t)std::max<long long>(p.slice_words, 1);
    const size_t per_slice_max = std::max<size_t>(1, kPmGlobalScratch / p.slice_bytes);
    // warp kernel: up to 8 warps per CTA, as many resident CTAs as fit, no more teams than rows
    const size_t W = std::min<size_t>(kPmThreads / 32, limit / p.slice_bytes);
    p.warp_global = W == 0;
    p.warp_block = p.warp_global ? 32 : (int)(32 * W);
    p.warp_smem = p.warp_global ? 0 : W * p.slice_bytes;
    size_t teams = std::max<size_t>(1, W);
    int occ = 1;
    if (!p.warp_global)
        GP_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gp_placement_rows<false>, p.warp_block, p.warp_smem));
    size_t grid = std::max<size_t>(1, std::min<size_t>(((size_t)Q + teams - 1) / teams, sm * (size_t)std::max(occ, 1)));
    if (p.warp_global) grid = std::min(grid, per_slice_max);
    p.warp_grid = (int)grid;
    // CTA kernel: one slice per CTA
    p.cta_global = p.slice_bytes > limit;
    p.cta_smem = p.cta_global ? 0 : p.slice_bytes;
    occ = 1;
    if (!p.cta_global) GP_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gp_placement_rows<true>, kPmThreads, p.cta_smem));
    grid = std::max<size_t>(1, std::min<size_t>((size_t)Q, sm * (size_t)std::max(occ, 1)));
    if (p.cta_global) grid = std::min(grid, per_slice_max);
    p.cta_grid = (int)grid;
    p.global_slices = std::max<size_t>(p.warp_global ? (size_t)p.warp_grid : 0, p.cta_global ? (size_t)p.cta_grid : 0);
    return GP_OK;
}

// the rows kernels and the finisher on st; in's arrays set, the scratch pieces taken from ar (reserved)
static gp_status pm_launch(gp_ctx* c, PmIn in, const PmPlan& p, gp_placement_record* out, int32_t* status, int32_t* bits, cudaStream_t st) {
    in.bitmap_words = p.bitmap_words;
    in.slice_words = p.slice_words;
    in.state = c->metricstate.as<PmState>();
    PmIn w = in, t = in;
    if (!p.warp_global) w.gslices = nullptr;
    if (!p.cta_global) t.gslices = nullptr;
    gp_placement_rows<false><<<p.warp_grid, p.warp_block, p.warp_smem, st>>>(w, out);
    gp_placement_rows<true><<<p.cta_grid, kPmThreads, p.cta_smem, st>>>(t, out);
    gp_placement_finish<<<1, 32, 0, st>>>(in.state, status, bits);
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// checks that need no array contents
static gp_status pm_check(gp_ctx* c, const gp_apps* a, const gp_results* r, int32_t N, const int32_t* zone, int32_t Z, const int32_t* ig,
                          int32_t G, const void* out, const char* who) {
    if (!a || !r || a->n_apps < 0 || N < 0 || Z < 0) return fail(c, GP_ERR_INVALID, who, "NULL apps/placed or a negative size");
    if (Z > std::max(N, 1)) return fail(c, GP_ERR_INVALID, who, "n_metric_zones above max(n_nodes, 1)");
    if (N > 0 && !zone) return fail(c, GP_ERR_INVALID, who, "metric_zone is NULL");
    if (ig && G < 1) return fail(c, GP_ERR_INVALID, who, "n_instance_groups must be >= 1");
    if (a->n_apps > 0 && (!out || !a->exe_count || !r->driver_node)) return fail(c, GP_ERR_INVALID, who, "missing app/result arrays");
    if (r->executor_nodes_cap < 0 || (r->executor_nodes_cap > 0 && !r->executor_nodes))
        return fail(c, GP_ERR_INVALID, who, "executor_nodes is NULL or executor_nodes_cap negative");
    return GP_OK;
}

extern "C" {

gp_status gp_placement_metrics(gp_ctx* c, const gp_apps* a, const gp_results* placed, int32_t N, const int32_t* zone, int32_t Z,
                               const int32_t* ig, int32_t G, gp_placement_record* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    const char* who = "gp_placement_metrics";
    GP_TRY(pm_check(c, a, placed, N, zone, Z, ig, G, out, who));
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    // host pass: offsets, exe_count, and the ExecutorNodes range each placed row reads
    std::vector<int64_t>& off = c->host_off;
    off.resize((size_t)Q + 1);
    int64_t acc = 0, used = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int32_t k = a->exe_count[i];
        if (k < 0) return fail(c, GP_ERR_INVALID, who, "negative exe_count");
        if (k > kPmMaxCount) return fail(c, GP_ERR_UNREPRESENTABLE, who, "exe_count above 2^24");
        off[(size_t)i] = a->exec_out_off ? a->exec_out_off[i] : acc;
        acc += k;
        if (placed->driver_node[i] < 0) continue;
        if (off[(size_t)i] < 0 || off[(size_t)i] > placed->executor_nodes_cap - k)
            return fail(c, GP_ERR_CAPACITY, who, "offsets exceed executor_nodes_cap");
        used = std::max<int64_t>(used, off[(size_t)i] + k);
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    PmPlan p;
    GP_TRY(pm_plan(c, N, Z, Q, p));
    GP_CUDA(c, c->metricstate.reserve(sizeof(PmState)));
    GP_CUDA(c, cudaMemsetAsync(c->metricstate.p, 0, sizeof(PmState), st));
    const size_t q = (size_t)Q, n = (size_t)N;
    const bool grouped = ig && a->group;
    Arena ar{c->metricbuf, st};
    const auto cnt = ar.take<int32_t>(q), grp = ar.take<int32_t>(grouped ? q : 0), drv = ar.take<int32_t>(q);
    const auto offp = ar.take<int64_t>(q + 1);
    const auto exe = ar.take<int32_t>((size_t)used);
    const auto zn = ar.take<int32_t>(n), igp = ar.take<int32_t>(ig ? n : 0);
    const auto rec = ar.take<gp_placement_record>(q);
    const auto word = ar.take<int32_t>(2);
    const auto lr = ar.take<int32_t>(q);
    const auto sl = ar.take<uint32_t>(p.global_slices * (size_t)p.slice_words);
    ar.reserve();
    PmIn in{};
    in.count = ar.put(cnt, a->exe_count);
    in.group = grouped ? ar.put(grp, a->group) : nullptr;
    in.driver = ar.put(drv, placed->driver_node);
    in.off = ar.put(offp, off.data());
    in.exec = used > 0 ? ar.put(exe, placed->executor_nodes) : ar.ptr(exe);
    in.cap = used;                                              // rows were checked against executor_nodes_cap above
    in.zone = ar.put(zn, zone);
    in.ig = ig ? ar.put(igp, ig) : nullptr;
    in.n_apps = Q; in.n_nodes = N; in.n_zones = Z; in.n_ig = ig ? G : 1;
    in.long_rows = ar.ptr(lr);
    in.gslices = ar.ptr(sl);
    GP_TRY(ar.check(c));
    int32_t* d_word = ar.ptr(word);
    GP_TRY(pm_launch(c, in, p, ar.ptr(rec), d_word, d_word + 1, st));
    int32_t hw[2] = {0, 0};
    std::vector<gp_placement_record>& recs = c->pm_records;      // a refused call writes no record into `out`
    recs.resize(q);
    ar.get(hw, word);
    ar.get(recs.data(), rec);
    GP_TRY(ar.sync(c));
    GP_TRY(refuse(c, hw[1], kPmRefusals, who));
    std::memcpy(out, recs.data(), sizeof(gp_placement_record) * q);
    return GP_OK;
}

gp_status gp_placement_metrics_device(gp_ctx* c, const gp_apps* da, const gp_results* dp, int32_t N, const int32_t* zone, int32_t Z,
                                      const int32_t* ig, int32_t G, gp_placement_record* dout, int32_t* dev_status, void* stream) {
    if (!enter(c)) return GP_ERR_INVALID;
    const char* who = "gp_placement_metrics_device";
    GP_TRY(pm_check(c, da, dp, N, zone, Z, ig, G, dout, who));
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
    const int32_t Q = da->n_apps;
    if (Q == 0) {
        if (dev_status) GP_CUDA(c, cudaMemsetAsync(dev_status, 0, sizeof(int32_t), st));
        return GP_OK;
    }
    PmPlan p;
    GP_TRY(pm_plan(c, N, Z, Q, p));
    GP_CUDA(c, c->metricstate.reserve(sizeof(PmState)));
    GP_CUDA(c, cudaMemsetAsync(c->metricstate.p, 0, sizeof(PmState), st));
    const size_t q = (size_t)Q;
    Arena ar{c->metricbuf, st};
    const auto offp = ar.take<int64_t>(da->exec_out_off ? 0 : q + 1);
    const auto lr = ar.take<int32_t>(q);
    const auto sl = ar.take<uint32_t>(p.global_slices * (size_t)p.slice_words);
    ar.reserve();
    GP_TRY(ar.check(c));
    PmIn in{};
    in.count = da->exe_count;
    in.group = ig ? da->group : nullptr;
    in.driver = dp->driver_node;
    in.exec = dp->executor_nodes;
    in.cap = dp->executor_nodes_cap;
    in.zone = zone;
    in.ig = ig;
    in.n_apps = Q; in.n_nodes = N; in.n_zones = Z; in.n_ig = ig ? G : 1;
    in.long_rows = ar.ptr(lr);
    in.gslices = ar.ptr(sl);
    if (da->exec_out_off) {
        in.off = da->exec_out_off;
    } else {
        int64_t* o = ar.ptr(offp);
        gp_placement_offsets<<<1, kPmThreads, 0, st>>>(da->exe_count, Q, o);
        in.off = o;
    }
    return pm_launch(c, in, p, dout, dev_status, nullptr, st);
}

}  // extern "C"
