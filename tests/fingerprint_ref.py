"""shape_fingerprint (csrc/gangpack_kernels.cuh) in plain Python integers, the two ways the kernels key it, and solvers that
build colliding requests.

Before its finalizer the fingerprint is  a K1 ^ (b + C2) K2 ^ (c + C3) K3  mod 2^64, and the finalizer (xorshift, odd
multiply, xorshift) is a bijection, so two tuples with the same pre-finalizer value collide in all 64 bits.  K1, K2 and K3
are odd, so any one dimension can be solved for once the other two are chosen; the solution is a valid quantity (< 2^61)
about one time in eight.

- gp_decide_tables interns executor requests by fingerprint(e0, e1, e2) and driver requests by
  fingerprint(d0 ^ DRIVER_SALT, d1, d2) in tables of SLOTS slots, PROBES linear probes from the home slot fp % SLOTS.
- gp_cc_intern (the unschedulable-pod marker) chains three: F(F(F(e0, e1, e2), d0, d1), d2, g) for the row
  (d0, d1, d2, e0, e1, e2) of class g.
"""
M64 = (1 << 64) - 1
K1, K2, K3 = 0x9E3779B97F4A7C15, 0x94D049BB133111EB, 0xD6E8FEB86659FD93
C2, C3 = 0xBF58476D1CE4E5B9, 0x2545F4914F6CDD1D
MIX = 0xBF58476D1CE4E5B9
DRIVER_SALT = 0x5bd1e995
MAX_QUANTITY = 1 << 61
SLOTS, PROBES, MAX_SHAPES = 1024, 16, 64          # kShapeSlots, kShapeProbes, kMaxShapes (gangpack_tables.cuh)
K = (K1, K2, K3)
ADD = (0, C2, C3)


def _term(d, v):
    return (((v + ADD[d]) & M64) * K[d]) & M64


def _pre(a, b, c):
    return _term(0, a & M64) ^ _term(1, b & M64) ^ _term(2, c & M64)


def fingerprint(a, b, c):
    """gp::shape_fingerprint; arguments are int64 values (negative ones wrap as in the kernel's casts)"""
    z = _pre(a, b, c)
    z ^= z >> 29
    z = (z * MIX) & M64
    z ^= z >> 32
    return z or 1


def driver_fingerprint(d0, d1, d2):
    return fingerprint(d0 ^ DRIVER_SALT, d1, d2)


def marker_fingerprint(row, g):
    """row = (drv cpu, mem, gpu, exe cpu, mem, gpu), g = its class (node group, -1 = every node, or affinity id)"""
    h = fingerprint(row[3], row[4], row[5])
    h = fingerprint(h, row[0], row[1])
    return fingerprint(h, row[2], g)


def _solve(target, d, rest):
    """the value v of dimension d with _term(d, v) ^ rest == target (mod 2^64)"""
    return ((((target ^ rest) * pow(K[d], -1, 1 << 64)) & M64) - ADD[d]) & M64


def collide(x, free_dim, others):
    """A tuple y != x with fingerprint(*y) == fingerprint(*x): dimension free_dim solved, the other two taken from `others`
    in dimension order.  None when the solution is not below 2^61."""
    y = list(others)
    y.insert(free_dim, 0)
    rest = 0
    for d in range(3):
        if d != free_dim:
            rest ^= _term(d, y[d])
    y[free_dim] = _solve(_pre(*x), free_dim, rest)
    y = tuple(y)
    return y if y[free_dim] < MAX_QUANTITY and y != tuple(x) else None


def collide_driver(x, free_dim, others):
    """collide() for driver requests (the salted first dimension)"""
    salt = lambda t: (t[0] ^ DRIVER_SALT,) + tuple(t[1:])
    o = list(others)
    if free_dim != 0:
        o[0] ^= DRIVER_SALT
    y = collide(salt(x), free_dim, o)
    return None if y is None else salt(y)


def collide_marker(x, gx, y, gy):
    """Row y with its driver gpu (index 2) solved so that marker_fingerprint(y, gy) == marker_fingerprint(x, gx); y's other
    fields are kept.  None when the solution is not below 2^61 or the rows are equal."""
    hx = fingerprint(fingerprint(x[3], x[4], x[5]), x[0], x[1])
    hy = fingerprint(fingerprint(y[3], y[4], y[5]), y[0], y[1])
    v = _solve(_pre(hx, x[2], gx), 1, _term(0, hy) ^ _term(2, gy & M64))
    out = tuple(y[:2]) + (v,) + tuple(y[3:])
    return out if v < MAX_QUANTITY and (out, gy) != (tuple(x), gx) else None


def home(fp):
    return fp & (SLOTS - 1)


def same_home(n, slot, driver=False, base=(1000, 1 << 30, 0), step=1 << 20):
    """n distinct requests base + (0, j step, 0) whose (driver) fingerprints have home slot `slot`"""
    f = driver_fingerprint if driver else fingerprint
    out, j = [], 0
    while len(out) < n:
        t = (base[0], base[1] + j * step, base[2])
        if home(f(*t)) == slot:
            out.append(t)
        j += 1
    return out


def distinct_homes(n, driver=False, base=(1000, 1 << 30, 0), step=1 << 20):
    """n requests base + (0, j step, 0) with pairwise distinct home slots: each is interned in its home slot, whatever the
    claim order"""
    f = driver_fingerprint if driver else fingerprint
    out, seen, j = [], set(), 0
    while len(out) < n:
        t = (base[0], base[1] + j * step, base[2])
        h = home(f(*t))
        if h not in seen:
            seen.add(h)
            out.append(t)
        j += 1
    return out


def window(slot):
    """the slots a request with home `slot` probes, in order"""
    return [(slot + p) % SLOTS for p in range(PROBES)]


# ---- the crafted sets of the GPU tests --------------------------------------------------------------------------------
GI, MI = 1 << 30, 1 << 20
HUGE = 1 << 50                      # a solved dimension at least this large exceeds every node of the tests


def _first(solver, x, free_dim, others_of_j):
    for j in range(1, 4096):
        y = solver(x, free_dim, others_of_j(j))
        if y is not None and y[free_dim] >= HUGE:
            return y
    raise AssertionError("no colliding tuple found")


def executor_pairs():
    """[(X, Y)]: realistic executor requests X and colliding Y with cpu, memory and gpu solved in turn; Y fits no node"""
    xs = [(1000, 4 * GI, 0), (2000, 2 * GI, 0), (1500, 3 * GI, 0)]
    others = [lambda j: (j * 256 * MI, 0), lambda j: (250 * j, 0), lambda j: (1500, 3 * GI + j * 128 * MI)]
    return [(x, _first(collide, x, d, others[d])) for d, x in enumerate(xs)]


def driver_pair():
    """(X, Y): a realistic driver request and a colliding one (memory solved) that fits no node"""
    x = (1000, 2 * GI, 0)
    return x, _first(collide_driver, x, 1, lambda j: (1000 + 250 * j, 0))


def marker_rows():
    """(A, B, C, ga, gc): marker rows (drv cpu, mem, gpu, exe cpu, mem, gpu).  A is realistic; B collides with A, both of
    class 0, and differs in its driver memory and its solved driver gpu; C, of class gc, has A's requests but its solved
    driver gpu and collides with A of class ga.  B and C fit no node.  (With equal other fields C's solution depends on the
    two classes alone, so they are searched for.)"""
    solved = lambda r: r is not None and r[2] >= HUGE
    a = (1000, GI, 0, 1000, GI, 0)
    b = next(r for r in (collide_marker(a, 0, a[:1] + (a[1] + j * MI,) + a[2:], 0) for j in range(1, 4096)) if solved(r))
    ga, gc = next((x, y) for x in range(8) for y in range(8) if x != y and solved(collide_marker(a, x, a, y)))
    return a, b, collide_marker(a, ga, a, gc), ga, gc


def full_window_sets():
    """17 executor and 17 driver requests with home slot 1020 (the window wraps to slot 11); and 16 executor requests with
    home slot 1020 plus one with home slot 1023"""
    ex = same_home(17, 1020)
    dr = same_home(17, 1020, driver=True, base=(500, GI, 0))
    mixed = same_home(16, 1020, base=(2000, GI, 0)) + same_home(1, 1023, base=(2000, GI, 0))
    return ex, dr, mixed


def shape_count_sets():
    """executor request sets of 64 and 65 shapes and driver request sets of 64, 65 and 300 shapes, distinct home slots"""
    ex = distinct_homes(65, base=(1000, GI, 0), step=64 * MI)
    dr = distinct_homes(300, driver=True, base=(500, GI // 2, 0), step=4 * MI)
    return {"exec64": ex[:64], "exec65": ex, "drv64": dr[:64], "drv65": dr[:65], "drv300": dr}
