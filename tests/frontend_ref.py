"""The snapshot front end in Python integers: availability from reservations (NodeSchedulingMetadataForNodes and the
first-fit availability of rescheduleExecutor) and the node priority orders of NodeSorter.PotentialNodes, as the library
documents them in include/gangpack.h.  Every quantity is a Python int, so no sum or difference has a bound: this is what the
device kernels must equal wherever their answer is representable, and what tells a wrapped answer from a right one.

Columns are plain sequences (lists or anything iterable of ints); None stands for an absent optional column."""

LIMIT = 1 << 61


def in_domain(x):
    """the exact-int64 domain of the library: |x| < 2^61"""
    return -LIMIT < x < LIMIT


def _col(c, n):
    return [0] * n if c is None else [int(x) for x in c]


def availability(alloc, overhead, res_node, res):
    """alloc / overhead / res: (cpu, mem, gpu) triples of columns (overhead, or any single column but alloc's and res's cpu
    and mem, may be None = 0); res_node[r]: node index of reservation r, rows outside [0, n) are ignored.
    -> (avail, sched, first_fit), each three lists of n Python ints:
         avail     = alloc - (sum of reservations + overhead)
         sched     = alloc - overhead
         first_fit = alloc - (sum of reservations + overhead * (2 if the node has a reservation row, whatever its
                     resources, else 1))"""
    n = len(alloc[0])
    al = [_col(alloc[d] if d < len(alloc) else None, n) for d in range(3)]
    ov = [_col(overhead[d] if overhead is not None and d < len(overhead) else None, n) for d in range(3)]
    rn = [int(x) for x in res_node]
    rs = [_col(res[d] if d < len(res) else None, len(rn)) for d in range(3)]
    usage = [[0] * n for _ in range(3)]
    has = [False] * n
    for r, node in enumerate(rn):
        if 0 <= node < n:
            has[node] = True
            for d in range(3):
                usage[d][node] += rs[d][r]
    avail = [[al[d][i] - (usage[d][i] + ov[d][i]) for i in range(n)] for d in range(3)]
    sched = [[al[d][i] - ov[d][i] for i in range(n)] for d in range(3)]
    first_fit = [[al[d][i] - (usage[d][i] + ov[d][i] * (2 if has[i] else 1)) for i in range(n)] for d in range(3)]
    return avail, sched, first_fit


def usage_sums(n, res_node, res):
    """per node and dimension, the sum of the reservations that count (for the domain checks of the tests)"""
    rn = [int(x) for x in res_node]
    rs = [_col(res[d] if d < len(res) else None, len(rn)) for d in range(3)]
    usage = [[0] * n for _ in range(3)]
    for r, node in enumerate(rn):
        if 0 <= node < n:
            for d in range(3):
                usage[d][node] += rs[d][r]
    return usage


def zone_totals(avail_cpu, avail_mem, zone_id, n_zones):
    """-> [(sum of memory, sum of cpu)] per zone id; an id without nodes totals (0, 0)"""
    tot = [[0, 0] for _ in range(n_zones)]
    if zone_id is not None:
        for c, m, z in zip(avail_cpu, avail_mem, zone_id):
            tot[z][0] += int(m)
            tot[z][1] += int(c)
    return [tuple(t) for t in tot]


def zone_totals_tied(avail_cpu, avail_mem, zone_id, n_zones):
    """True when two zones that have nodes share their (memory, cpu) totals: the one case the reference's zone order leaves
    open (the library orders such zones by id)"""
    if zone_id is None or n_zones <= 1:
        return False
    tot = zone_totals(avail_cpu, avail_mem, zone_id, n_zones)
    used = sorted({int(z) for z in zone_id})
    return len({tot[z] for z in used}) < len(used)


def zone_priority(avail_cpu, avail_mem, zone_id, n_zones):
    """priority of every zone id = its rank by (memory total, cpu total, id) over ALL n_zones ids"""
    tot = zone_totals(avail_cpu, avail_mem, zone_id, n_zones)
    prio = [0] * n_zones
    for rank, z in enumerate(sorted(range(n_zones), key=lambda z: (tot[z][0], tot[z][1], z))):
        prio[z] = rank
    return prio


def node_keys(avail_cpu, avail_mem, zone_id=None, n_zones=1):
    """-> [(zone priority, memory, cpu)] per node"""
    n = len(avail_cpu)
    if zone_id is None or n_zones <= 1:
        return [(0, int(avail_mem[i]), int(avail_cpu[i])) for i in range(n)]
    prio = zone_priority(avail_cpu, avail_mem, zone_id, n_zones)
    return [(prio[int(zone_id[i])], int(avail_mem[i]), int(avail_cpu[i])) for i in range(n)]


def priority_order(avail_cpu, avail_mem, zone_id=None, n_zones=1, name_rank=None):
    """every node in ascending (zone priority, memory, cpu, name rank) order; name_rank None = index order"""
    keys = node_keys(avail_cpu, avail_mem, zone_id, n_zones)
    nr = range(len(keys)) if name_rank is None else [int(x) for x in name_rank]
    return sorted(range(len(keys)), key=lambda i: (keys[i], nr[i]))


def label_sort(order, label_rank):
    """stable re-sort by label rank, unknown (-1) last; None = not configured"""
    if label_rank is None:
        return list(order)
    return sorted(order, key=lambda i: (1, 0) if label_rank[i] < 0 else (0, int(label_rank[i])))


def potential_nodes(avail_cpu, avail_mem, zone_id=None, n_zones=1, name_rank=None, cand=None, unsched=None, ready=None,
                    lr_d=None, lr_e=None):
    """-> (driver order, executor order) as lists of node indices: the priority order restricted to the driver candidates /
    to the schedulable and ready nodes, each re-sorted stably by its label rank when one is configured"""
    order = priority_order(avail_cpu, avail_mem, zone_id, n_zones, name_rank)
    drv = [i for i in order if cand is None or cand[i]]
    exe = [i for i in order if not (unsched is not None and unsched[i]) and (ready is None or ready[i])]
    return label_sort(drv, lr_d), label_sort(exe, lr_e)


def undefined_ties(order, keys, gpu):
    """adjacent pairs of `order` with equal (zone priority, memory, cpu) and different gpu"""
    if gpu is None:
        return 0
    return sum(1 for a, b in zip(order, order[1:]) if keys[a] == keys[b] and int(gpu[a]) != int(gpu[b]))
