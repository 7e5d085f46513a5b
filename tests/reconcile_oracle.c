/* reconcile_oracle.c -- literal, string-keyed restatement of the failover reconciler's node choice (TEST INFRASTRUCTURE ONLY;
 * compiled by tests/reconcile_ref.py and linked into the C++ host-layer test, never into libgangpack.so).
 *
 * EXT = internal/extender, LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg.  Every map of the reference is a
 * string-keyed hash map here, every quantity an exact __int128 (the reference's resource.Quantity has no int64 bound; a value
 * leaving |v| < 2^61 is reported, which is where gp_reconcile_find_nodes refuses).
 *
 *   availableResourcesPerInstanceGroup   EXT/failover.go:286-323
 *   syncResourceReservations (stale driver branch, charge of :159)   EXT/failover.go:136-160
 *   constructResourceReservation         EXT/failover.go:348-390
 *   findNodes                            EXT/failover.go:409-436
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef __int128 q_t;
typedef struct { q_t v[3]; } res_t;                 /* Resources{CPU, Memory, NvidiaGPU} */

static res_t rz(void) { res_t r; memset(&r, 0, sizeof r); return r; }
static void radd(res_t* a, const res_t* b) { for (int d = 0; d < 3; ++d) a->v[d] += b->v[d]; }          /* Resources.Add */
static void rsub(res_t* a, const res_t* b) { for (int d = 0; d < 3; ++d) a->v[d] -= b->v[d]; }          /* Resources.Sub */
static int rgt(const res_t* a, const res_t* b) {                                                         /* Resources.GreaterThan */
    return a->v[0] > b->v[0] || a->v[1] > b->v[1] || a->v[2] > b->v[2];
}

/* ---- string-keyed map (open addressing, FNV-1a) ------------------------------------------------------------------------- */
typedef struct { const char** key; res_t* val; size_t cap; } smap;
static uint64_t fnv(const char* s) { uint64_t h = 1469598103934665603ull; while (*s) { h ^= (unsigned char)*s++; h *= 1099511628211ull; } return h; }
static void smap_init(smap* m, size_t n) {
    m->cap = 16; while (m->cap < 2 * n + 16) m->cap <<= 1;
    m->key = calloc(m->cap, sizeof(char*)); m->val = calloc(m->cap, sizeof(res_t));
}
static void smap_free(smap* m) { free(m->key); free(m->val); }
static res_t* smap_get(smap* m, const char* k) {           /* NULL when absent */
    for (size_t i = fnv(k) & (m->cap - 1);; i = (i + 1) & (m->cap - 1)) {
        if (!m->key[i]) return NULL;
        if (!strcmp(m->key[i], k)) return &m->val[i];
    }
}
static size_t smap_slot(smap* m, const char* k, int* created) {   /* slot of k, created as Zero() */
    for (size_t i = fnv(k) & (m->cap - 1);; i = (i + 1) & (m->cap - 1)) {
        if (!m->key[i]) { m->key[i] = k; m->val[i] = rz(); *created = 1; return i; }
        if (!strcmp(m->key[i], k)) { *created = 0; return i; }
    }
}
static res_t* smap_put(smap* m, const char* k) { int c; return &m->val[smap_slot(m, k, &c)]; }

static const int64_t* g_creation;
/* sort.Slice(nodes, nodes[j].CreationTimestamp.Before(&nodes[i].CreationTimestamp)) (:292-294).  The node table is the lister's
 * order; ties keep it (a newest-first lister order comes back unchanged from Go 1.19's pdqsort, DESIGN §2.3). */
static int newest_first(const void* a, const void* b) {
    const int32_t i = *(const int32_t*)a, j = *(const int32_t*)b;
    if (g_creation[i] != g_creation[j]) return g_creation[i] > g_creation[j] ? -1 : 1;
    return i < j ? -1 : (i > j);
}

static int out_of_domain(q_t v) { const q_t lim = (q_t)1 << 61; return v >= lim || v <= -lim; }

/* Returns 0, or 1 when a charged availability left |v| < 2^61 (outputs are still the exact result, truncated to int64).
 *   nodes        names[n], allocatable, instance-group label value (NULL = label missing = ""), unschedulable, ready, creation
 *   overhead     GetOverhead per node (NULL columns = 0)
 *   rows         every RR reservation and soft reservation: node name (need not be in the table) and resources
 *   drivers      in processing order: the group FindInstanceGroupFromPodSpec returns (NULL = ""), executor resources,
 *                MinExecutorCount and the number of running executors
 *   placed[i]    -1 when constructResourceReservation errs ("instance group not found"), else len(reservedNodeNames)
 *   out_nodes    reservedNodeNames as node-table indices, at off[i] = sum over j < i of max(0, Min_j - min(running_j, Min_j))
 *   avail_*      [n] availability after the loop (nodes of no group: allocatable - usage, never charged) */
int orc_reconcile_find_nodes(int32_t n, const char** names, const int64_t* alloc_cpu, const int64_t* alloc_mem, const int64_t* alloc_gpu,
                             const char** group_label, const uint8_t* unschedulable, const uint8_t* ready, const int64_t* creation,
                             const int64_t* over_cpu, const int64_t* over_mem, const int64_t* over_gpu,
                             int64_t n_rows, const char** row_node, const int64_t* row_cpu, const int64_t* row_mem, const int64_t* row_gpu,
                             int32_t q, const char** drv_group, const int64_t* exe_cpu, const int64_t* exe_mem, const int64_t* exe_gpu,
                             const int32_t* min_count, const int32_t* running,
                             int32_t* placed, int32_t* out_nodes, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu) {
    int bad = 0;
    /* :292-294 */
    int32_t* sorted = malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    for (int32_t i = 0; i < n; ++i) sorted[i] = i;
    g_creation = creation;
    qsort(sorted, (size_t)n, sizeof(int32_t), newest_first);
    /* :296-314: schedulableNodes[instanceGroup(n.Labels[label])] = append(...), unschedulable / not-ready skipped; the groups are
     * kept as one list of distinct label values with, per value, the nodes in the sorted order */
    const char** gname = malloc(sizeof(char*) * (size_t)(n > 0 ? n : 1));
    int32_t* gsize = calloc((size_t)(n > 0 ? n : 1), sizeof(int32_t));
    int32_t* gnodes = malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));   /* node -> group slot, -1 = skipped */
    int32_t ng = 0;
    for (int32_t s = 0; s < n; ++s) {
        const int32_t v = sorted[s];
        gnodes[v] = -1;
        if (unschedulable && unschedulable[v]) continue;                 /* :297-299 */
        if (ready && !ready[v]) continue;                                /* :301-309 */
        const char* ig = group_label[v] ? group_label[v] : "";           /* :312: a missing label is "" */
        int32_t g = 0;
        while (g < ng && strcmp(gname[g], ig)) ++g;
        if (g == ng) gname[ng++] = ig;
        gnodes[v] = g;
        ++gsize[g];
    }
    /* orderedNodes[g]: per group the nodes in the sorted order */
    int32_t* goff = calloc((size_t)ng + 1, sizeof(int32_t));
    for (int32_t g = 0; g < ng; ++g) goff[g + 1] = goff[g] + gsize[g];
    int32_t* gorder = malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    int32_t* fill = calloc((size_t)ng + 1, sizeof(int32_t));
    for (int32_t s = 0; s < n; ++s) {
        const int32_t v = sorted[s];
        if (gnodes[v] >= 0) gorder[goff[gnodes[v]] + fill[gnodes[v]]++] = v;
    }
    /* :315-317 usages = UsageForNodes(rrs); usages.Add(overhead); usages.Add(softReservationOverhead) */
    smap usage;
    smap_init(&usage, (size_t)n + (size_t)n_rows);
    for (int64_t r = 0; r < n_rows; ++r) {
        res_t x = rz();
        x.v[0] = row_cpu[r]; x.v[1] = row_mem[r]; x.v[2] = row_gpu ? row_gpu[r] : 0;
        radd(smap_put(&usage, row_node[r]), &x);
    }
    for (int32_t v = 0; v < n; ++v) {
        res_t o = rz();
        o.v[0] = over_cpu ? over_cpu[v] : 0; o.v[1] = over_mem ? over_mem[v] : 0; o.v[2] = over_gpu ? over_gpu[v] : 0;
        radd(smap_put(&usage, names[v]), &o);
    }
    /* :318-321 availableResources[g] = AvailableForNodes(ns, usages) (LIB/resources/resources.go:45-56) */
    smap avail;
    smap_init(&avail, (size_t)n);
    for (int32_t v = 0; v < n; ++v) {
        res_t* a = smap_put(&avail, names[v]);
        a->v[0] = alloc_cpu[v]; a->v[1] = alloc_mem[v]; a->v[2] = alloc_gpu ? alloc_gpu[v] : 0;
        res_t* u = smap_get(&usage, names[v]);
        if (u) rsub(a, u);
    }
    /* the stale drivers (:70-76, in the given order) */
    smap reserved;                                      /* findNodes' map, emptied slot by slot after each driver */
    smap_init(&reserved, (size_t)n);
    size_t* touched = malloc(sizeof(size_t) * (size_t)(n > 0 ? n : 1));
    int64_t off = 0;
    for (int32_t i = 0; i < q; ++i) {
        const int32_t run = running[i] < min_count[i] ? running[i] : min_count[i];          /* executorsUpToMin, :141-143 */
        const int32_t k = min_count[i] - run;                                                /* :366 */
        const int64_t base = off;
        off += k > 0 ? k : 0;
        /* constructResourceReservation :358-362: the group must be in orderedNodes (checked before the count) */
        const char* ig = drv_group[i] ? drv_group[i] : "";
        int32_t g = 0;
        while (g < ng && strcmp(gname[g], ig)) ++g;
        if (g == ng) { placed[i] = -1; continue; }
        placed[i] = 0;
        if (k <= 0) continue;                                                                /* :367: reservedResources nil */
        res_t exe = rz();
        exe.v[0] = exe_cpu[i]; exe.v[1] = exe_mem[i]; exe.v[2] = exe_gpu ? exe_gpu[i] : 0;
        /* findNodes :412-436 */
        size_t n_touched = 0;
        int32_t got = 0;
        for (int32_t s = goff[g]; s < goff[g + 1] && got < k; ++s) {
            const char* nm = names[gorder[s]];
            int created;
            const size_t slot = smap_slot(&reserved, nm, &created);                          /* :421-423 */
            if (created) touched[n_touched++] = slot;
            res_t* rn = &reserved.val[slot];
            const res_t* an = smap_get(&avail, nm);
            for (;;) {
                radd(rn, &exe);                                                              /* :425 */
                if (rgt(rn, an)) break;                                                      /* :426-428 */
                out_nodes[base + got++] = gorder[s];                                         /* :429 */
                if (got == k) break;                                                         /* :430-432 */
            }
        }
        placed[i] = got;
        /* :159 r.availableResources[instanceGroup].Sub(reservedResources) */
        for (size_t t = 0; t < n_touched; ++t) {
            const size_t h = touched[t];
            res_t* an = smap_get(&avail, reserved.key[h]);
            rsub(an, &reserved.val[h]);
            for (int d = 0; d < 3; ++d) bad |= out_of_domain(an->v[d]);
        }
        for (size_t t = 0; t < n_touched; ++t) reserved.key[touched[t]] = NULL;
    }
    for (int32_t v = 0; v < n; ++v) {
        const res_t* a = smap_get(&avail, names[v]);
        if (avail_cpu) avail_cpu[v] = (int64_t)a->v[0];
        if (avail_mem) avail_mem[v] = (int64_t)a->v[1];
        if (avail_gpu) avail_gpu[v] = (int64_t)a->v[2];
    }
    smap_free(&usage); smap_free(&avail); smap_free(&reserved);
    free(touched); free(sorted); free(gname); free(gsize); free(gnodes); free(goff); free(gorder); free(fill);
    return bad;
}
