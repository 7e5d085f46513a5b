// gangpack_multi.cu -- one HOST process driving several GPUs of one box through the C ABI (include/gangpack.h, gp_multi_*).
//
// The reference is ONE process with a serial Predicate (internal/extender/resource.go:194-205, packer chosen once at
// cmd/server.go:145); a cgo host therefore needs a single handle that uses every GPU, not one process per device:
//   * one gp_ctx per device and one persistent worker thread per context (CUDA calls of different devices overlap);
//   * the snapshot goes to every device by direct H2D copies, each over the device's OWN PCIe link, in parallel;
//   * GP_MODE_INDEPENDENT (SURVEY 8e row 1): the queue is cut into one contiguous block per device; every device packs
//     its block and copies ITS placements straight into the caller's result buffers at the block's position -- no
//     gather through one GPU, no collective (the path has no exchange step);
//   * FIFO modes (SURVEY 8e row 2; per-group independence: internal/extender/sparkpods.go:61, resource.go:292-295):
//     whole instance groups are assigned to devices (longest-processing-time first on apps_g x nodes_g), every device
//     runs the queues of its groups in order against its copy of the snapshot, results are scattered back into queue
//     order; gp_multi_get_snapshot reads every node from the device that owns its group.
// Host code only: it calls the public gp_* entry points and launches no kernel of its own.
#include "gangpack.h"

#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

namespace {

struct Worker {
    gp_ctx* ctx = nullptr;
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    std::function<gp_status()> job;
    bool has_job = false, done = true, quit = false;
    gp_status result = GP_OK;

    void loop() {
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv.wait(lk, [&] { return has_job || quit; });
            if (quit) return;
            std::function<gp_status()> j = std::move(job);
            has_job = false;
            lk.unlock();
            const gp_status r = j();
            lk.lock();
            result = r;
            done = true;
            cv.notify_all();
        }
    }
    void submit(std::function<gp_status()> j) {
        std::lock_guard<std::mutex> lk(mu);
        job = std::move(j); has_job = true; done = false;
        cv.notify_all();
    }
    gp_status wait() {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return done; });
        return result;
    }
};

}  // namespace

struct gp_multi {
    std::vector<Worker*> w;
    std::string err;
    // snapshot facts kept on the host
    int32_t n_nodes = 0, n_groups = 0;
    std::vector<int32_t> node_group;       // [n_nodes] instance group of a node, -1 = in no order
    std::vector<int64_t> group_nodes;      // [n_groups] executor + driver candidates (cost model)
    std::vector<int32_t> owner;            // [n_groups] device index that ran the group's queue in the last FIFO batch
    bool have_snapshot = false;
};

static gp_status mfail(gp_multi* m, gp_status st, const std::string& msg) { m->err = msg; return st; }

// run f(device index) on every worker, first failure wins
static gp_status run_all(gp_multi* m, const std::function<gp_status(int)>& f) {
    const int n = (int)m->w.size();
    for (int d = 0; d < n; ++d) m->w[d]->submit([&f, d] { return f(d); });
    gp_status st = GP_OK;
    int bad = -1;
    for (int d = 0; d < n; ++d) {
        const gp_status r = m->w[d]->wait();
        if (r != GP_OK && st == GP_OK) { st = r; bad = d; }
    }
    if (st != GP_OK) m->err = "device " + std::to_string(bad) + ": " + gp_last_error(m->w[bad]->ctx);
    return st;
}

extern "C" {

gp_status gp_multi_create(gp_multi** out, const int32_t* devices, int32_t n_devices) {
    if (!out || n_devices < 1 || n_devices > 64) return GP_ERR_INVALID;
    *out = nullptr;
    gp_multi* m = new (std::nothrow) gp_multi();
    if (!m) return GP_ERR_INVALID;
    for (int32_t i = 0; i < n_devices; ++i) {
        gp_config cfg{};
        cfg.device = devices ? devices[i] : i;
        gp_ctx* c = nullptr;
        const gp_status st = gp_create(&c, &cfg);
        if (st != GP_OK) {
            for (Worker* w : m->w) { gp_destroy(w->ctx); delete w; }
            delete m;
            return st;                  // gp_last_error(NULL) describes it
        }
        Worker* w = new Worker();
        w->ctx = c;
        m->w.push_back(w);
    }
    for (Worker* w : m->w) w->th = std::thread([w] { w->loop(); });
    *out = m;
    return GP_OK;
}

void gp_multi_destroy(gp_multi* m) {
    if (!m) return;
    for (Worker* w : m->w) {
        { std::lock_guard<std::mutex> lk(w->mu); w->quit = true; }
        w->cv.notify_all();
        if (w->th.joinable()) w->th.join();
        gp_destroy(w->ctx);
        delete w;
    }
    delete m;
}

const char* gp_multi_last_error(const gp_multi* m) { return m ? m->err.c_str() : gp_last_error(nullptr); }
int32_t gp_multi_size(const gp_multi* m) { return m ? (int32_t)m->w.size() : 0; }
gp_ctx* gp_multi_ctx(gp_multi* m, int32_t i) { return (m && i >= 0 && i < (int32_t)m->w.size()) ? m->w[(size_t)i]->ctx : nullptr; }

gp_status gp_multi_set_snapshot(gp_multi* m, const gp_nodes* n) {
    if (!m) return GP_ERR_INVALID;
    if (!n || n->n_nodes < 0 || n->n_groups < 1 || !n->exec_off || !n->drv_off) return mfail(m, GP_ERR_INVALID, "gp_multi_set_snapshot: missing arrays or bad sizes");
    const gp_status st = run_all(m, [&](int d) { return gp_set_snapshot(m->w[(size_t)d]->ctx, n); });   // validates; N parallel H2D
    if (st != GP_OK) { m->have_snapshot = false; return st; }
    m->n_nodes = n->n_nodes; m->n_groups = n->n_groups;
    m->node_group.assign((size_t)n->n_nodes, -1);
    m->group_nodes.assign((size_t)n->n_groups, 0);
    for (int32_t g = 0; g < n->n_groups; ++g) {
        for (int32_t e = n->exec_off[g]; e < n->exec_off[g + 1]; ++e) m->node_group[(size_t)n->exec_order[e]] = g;
        for (int32_t e = n->drv_off[g]; e < n->drv_off[g + 1]; ++e) m->node_group[(size_t)n->drv_order[e]] = g;
        m->group_nodes[(size_t)g] = std::max<int64_t>(n->exec_off[g + 1] - n->exec_off[g], n->drv_off[g + 1] - n->drv_off[g]);
    }
    m->owner.assign((size_t)n->n_groups, 0);
    m->have_snapshot = true;
    return GP_OK;
}

gp_status gp_multi_group_owner(gp_multi* m, int32_t* owner) {
    if (!m || !owner) return GP_ERR_INVALID;
    if (!m->have_snapshot) return mfail(m, GP_ERR_NO_SNAPSHOT, "gp_multi_group_owner: no snapshot");
    std::memcpy(owner, m->owner.data(), sizeof(int32_t) * m->owner.size());
    return GP_OK;
}

gp_status gp_multi_get_snapshot(gp_multi* m, int64_t* cpu, int64_t* mem, int64_t* gpu) {
    if (!m) return GP_ERR_INVALID;
    if (!m->have_snapshot) return mfail(m, GP_ERR_NO_SNAPSHOT, "gp_multi_get_snapshot: no snapshot");
    const size_t N = (size_t)m->n_nodes, D = m->w.size();
    std::vector<int64_t> buf(3 * N * D);
    const gp_status st = run_all(m, [&](int d) {
        int64_t* b = buf.data() + 3 * N * (size_t)d;
        return gp_get_snapshot(m->w[(size_t)d]->ctx, b, b + N, b + 2 * N);
    });
    if (st != GP_OK) return st;
    for (size_t i = 0; i < N; ++i) {
        const int32_t g = m->node_group[i];
        const size_t d = g >= 0 ? (size_t)m->owner[(size_t)g] : 0;      // a node in no order is never charged: any copy
        const int64_t* b = buf.data() + 3 * N * d;
        if (cpu) cpu[i] = b[i];
        if (mem) mem[i] = b[N + i];
        if (gpu) gpu[i] = b[2 * N + i];
    }
    return GP_OK;
}

gp_status gp_multi_pack_batch(gp_multi* m, const gp_apps_wire* a, gp_algo algo, gp_mode mode, gp_results_wire* out) {
    if (!m) return GP_ERR_INVALID;
    if (!m->have_snapshot) return mfail(m, GP_ERR_NO_SNAPSHOT, "gp_multi_pack_batch: gp_multi_set_snapshot first");
    if (!a || !out || a->n_apps < 0) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: NULL apps/results");
    if ((a->quantity_bits != 64 && a->quantity_bits != 32) || (out->node_bits != 32 && out->node_bits != 16))
        return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: quantity_bits must be 64 or 32, node_bits 32 or 16");
    const int32_t q = a->n_apps;
    if (q == 0) return GP_OK;
    if (!a->drv_cpu || !a->drv_mem || !a->exe_cpu || !a->exe_mem || !a->exe_count || !out->driver_node)
        return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: missing app/result arrays");
    const int D = (int)m->w.size();
    const size_t es = a->quantity_bits == 64 ? 8 : 4, os = out->node_bits == 16 ? 2 : 4;
    auto col = [&](const void* p, size_t lo) -> const void* { return p ? static_cast<const char*>(p) + es * lo : nullptr; };

    if (mode == GP_MODE_INDEPENDENT) {
        // ---- contiguous block of the queue per device; ExecutorNodes base of every block from the counts ---------
        std::vector<int32_t> lo((size_t)D + 1);
        for (int d = 0; d <= D; ++d) lo[(size_t)d] = (int32_t)((int64_t)q * d / D);
        std::vector<int64_t> base((size_t)D + 1, 0);
        if (a->exec_out_off) {
            for (int d = 0; d <= D; ++d) base[(size_t)d] = a->exec_out_off[lo[(size_t)d]];
        } else {
            std::vector<int64_t> part((size_t)D, 0);
            run_all(m, [&](int d) {                                  // each worker sums its own block
                int64_t acc = 0;
                for (int32_t i = lo[(size_t)d]; i < lo[(size_t)d + 1]; ++i) acc += a->exe_count[i] > 0 ? a->exe_count[i] : 0;
                part[(size_t)d] = acc;
                return GP_OK;
            });
            for (int d = 0; d < D; ++d) base[(size_t)d + 1] = base[(size_t)d] + part[(size_t)d];
        }
        if (base[(size_t)D] > out->executor_nodes_cap) return mfail(m, GP_ERR_CAPACITY, "gp_multi_pack_batch: executor_nodes_cap too small");
        if (base[(size_t)D] > 0 && !out->executor_nodes) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: executor_nodes is NULL");
        const bool fused = algo != GP_MINIMAL_FRAGMENTATION;
        return run_all(m, [&](int d) -> gp_status {
            const size_t l = (size_t)lo[(size_t)d];
            const int32_t n = lo[(size_t)d + 1] - lo[(size_t)d];
            if (n == 0) return GP_OK;
            gp_apps_wire s = *a;
            s.n_apps = n;
            s.drv_cpu = col(a->drv_cpu, l); s.drv_mem = col(a->drv_mem, l); s.drv_gpu = col(a->drv_gpu, l);
            s.exe_cpu = col(a->exe_cpu, l); s.exe_mem = col(a->exe_mem, l); s.exe_gpu = col(a->exe_gpu, l);
            s.exe_count = a->exe_count + l;
            s.group = a->group ? a->group + l : nullptr;
            s.skip_if_no_fit = nullptr;
            std::vector<int64_t> rebased;
            if (fused) s.exec_out_off = nullptr;                    // derived on the device, relative to this block
            else {
                // minimal-fragmentation needs offsets: this block's, rebased to 0
                rebased.resize((size_t)n + 1);
                int64_t acc = 0;
                for (int32_t i = 0; i < n; ++i) { rebased[(size_t)i] = acc; acc += s.exe_count[i] > 0 ? s.exe_count[i] : 0; }
                rebased[(size_t)n] = acc;
                s.exec_out_off = rebased.data();
            }
            gp_results_wire r = *out;
            r.driver_node = out->driver_node + l;
            r.executor_nodes = out->executor_nodes ? static_cast<char*>(out->executor_nodes) + os * (size_t)base[(size_t)d] : nullptr;
            r.executor_nodes_cap = base[(size_t)d + 1] - base[(size_t)d];
            return gp_pack_batch_wire(m->w[(size_t)d]->ctx, &s, algo, mode, &r);
        });
    }

    // ---- FIFO modes: whole instance groups per device ------------------------------------------------------------
    if (out->node_bits != 32) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: FIFO modes emit int32 node indices");
    if (!a->exec_out_off) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: FIFO modes need exec_out_off");
    if (a->exec_out_off[q] > out->executor_nodes_cap) return mfail(m, GP_ERR_CAPACITY, "gp_multi_pack_batch: executor_nodes_cap too small");
    if (a->exec_out_off[q] > 0 && !out->executor_nodes) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: executor_nodes is NULL");
    const int32_t G = m->n_groups;
    std::vector<int64_t> apps_in((size_t)G, 0);
    for (int32_t i = 0; i < q; ++i) {
        const int32_t g = a->group ? a->group[i] : 0;
        if (g < 0 || g >= G) return mfail(m, GP_ERR_INVALID, "gp_multi_pack_batch: app group out of range");
        apps_in[(size_t)g]++;
    }
    {   // longest-processing-time first: cost of a group's queue ~ applications x nodes
        std::vector<int32_t> order((size_t)G);
        std::iota(order.begin(), order.end(), 0);
        auto cost = [&](int32_t g) { return apps_in[(size_t)g] * std::max<int64_t>(m->group_nodes[(size_t)g], 1); };
        std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return cost(x) > cost(y); });
        std::vector<int64_t> load((size_t)D, 0);
        for (int32_t g : order) {
            const int d = (int)(std::min_element(load.begin(), load.end()) - load.begin());
            m->owner[(size_t)g] = d;
            load[(size_t)d] += cost(g);
        }
    }
    const int64_t* off = a->exec_out_off;
    return run_all(m, [&](int d) -> gp_status {
        // gather this device's sub-queue (queue order preserved), run it, scatter the results back
        std::vector<int32_t> idx;
        idx.reserve((size_t)q / (size_t)D + 16);
        for (int32_t i = 0; i < q; ++i) if (m->owner[(size_t)(a->group ? a->group[i] : 0)] == d) idx.push_back(i);
        const size_t n = idx.size();
        if (n == 0) return GP_OK;
        std::vector<char> cols(6 * es * n);
        const void* src[6] = {a->drv_cpu, a->drv_mem, a->drv_gpu, a->exe_cpu, a->exe_mem, a->exe_gpu};
        for (int c = 0; c < 6; ++c) {
            if (!src[c]) continue;
            char* dst = cols.data() + (size_t)c * es * n;
            if (es == 8) { auto* s8 = static_cast<const int64_t*>(src[c]); auto* d8 = reinterpret_cast<int64_t*>(dst); for (size_t j = 0; j < n; ++j) d8[j] = s8[idx[j]]; }
            else { auto* s4 = static_cast<const int32_t*>(src[c]); auto* d4 = reinterpret_cast<int32_t*>(dst); for (size_t j = 0; j < n; ++j) d4[j] = s4[idx[j]]; }
        }
        std::vector<int32_t> cnt(n), grp(n), drv(n);
        std::vector<uint8_t> skip(n, 0);
        std::vector<int64_t> soff(n + 1);
        int64_t acc = 0;
        for (size_t j = 0; j < n; ++j) {
            const int32_t i = idx[j];
            cnt[j] = a->exe_count[i];
            grp[j] = a->group ? a->group[i] : 0;
            if (a->skip_if_no_fit) skip[j] = a->skip_if_no_fit[i];
            soff[j] = acc;
            acc += cnt[j] > 0 ? cnt[j] : 0;
        }
        soff[n] = acc;
        std::vector<int32_t> exe((size_t)acc + 1);
        gp_apps_wire s = *a;
        s.n_apps = (int32_t)n;
        s.drv_cpu = cols.data(); s.drv_mem = cols.data() + es * n; s.drv_gpu = a->drv_gpu ? cols.data() + 2 * es * n : nullptr;
        s.exe_cpu = cols.data() + 3 * es * n; s.exe_mem = cols.data() + 4 * es * n; s.exe_gpu = a->exe_gpu ? cols.data() + 5 * es * n : nullptr;
        s.exe_count = cnt.data(); s.group = grp.data(); s.skip_if_no_fit = a->skip_if_no_fit ? skip.data() : nullptr;
        s.exec_out_off = soff.data();
        gp_results_wire r{drv.data(), exe.data(), acc, 32, 0};
        const gp_status st = gp_pack_batch_wire(m->w[(size_t)d]->ctx, &s, algo, mode, &r);
        if (st != GP_OK) return st;
        int32_t* oe = static_cast<int32_t*>(out->executor_nodes);
        for (size_t j = 0; j < n; ++j) {
            const int32_t i = idx[j];
            out->driver_node[i] = drv[j];
            if (drv[j] >= 0 && cnt[j] > 0) std::memcpy(oe + off[i], exe.data() + soff[j], sizeof(int32_t) * (size_t)cnt[j]);
        }
        return GP_OK;
    });
}

}  // extern "C"
