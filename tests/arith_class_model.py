"""Model of the capacity arithmetic's class dispatch, in Python integers.

Every decision rests on cap(n) = min over dims of floor((avail - r) / e).  The kernels pick, per application, an
arithmetic class and per dimension a divider kind (csrc/gangpack_kernels.cuh: prep_dim, prep_fast32, pack_app;
csrc/gangpack_resched.cuh: make_dimdiv; csrc/gangpack_api.cu: shift_for, compact_pair).  This module restates those
choices and emulates each class's arithmetic bit for bit (32-bit words, multiply-high, funnel shift), so that the tests
can check every class against floor division and can tell which class a given application lands in.
"""
from __future__ import annotations

from collections import namedtuple

M32 = (1 << 32) - 1
M64 = (1 << 64) - 1
MAX_QUANTITY = 1 << 61
MAX_COUNT = 1 << 24

K_INF, K_MAGIC, K_SHIFT, K_SLOW = 0, 1, 2, 3

# divider kinds as the tests name them: kDivMagic is split into the power-of-two trick and a true odd divisor
INF, SHIFT, MAGIC2, MAGIC, SLOW = "inf", "shift", "magic2", "magic", "slow"
KINDS = (INF, SHIFT, MAGIC2, MAGIC, SLOW)
FAST32, FAST64, GENERAL = "fast32", "fast64", "general"
CLASSES = (FAST32, FAST64, GENERAL)

DimDiv = namedtuple("DimDiv", "magic e sh kind")


def kind_name(dv: DimDiv) -> str:
    if dv.kind == K_INF:
        return INF
    if dv.kind == K_SHIFT:
        return SHIFT
    if dv.kind == K_SLOW:
        return SLOW
    return MAGIC2 if dv.magic == 1 << 63 else MAGIC


def ctz(e: int) -> int:
    return (e & -e).bit_length() - 1


# ---- the dispatch ----------------------------------------------------------------------------------------------------
def shift_for(mx: int) -> int:
    """Smallest S with mx >> S < 2^32 (0 for mx <= 0): the compact view's shift."""
    if mx <= 0:
        return 0
    bits = mx.bit_length()
    return bits - 32 if bits > 32 else 0


def prep_dim(e: int, t: int, max_avail: int):
    """-> (DimDiv, fast): the division recipe of executor request e in dimension t (0 cpu, 1 mem, 2 gpu) and whether the
    dimension qualifies for the fast class against a snapshot whose largest availability is max_avail."""
    magic, sh, kind = 0, 0, K_INF
    if e > 0:
        sh = ctz(e)
        odd = e >> sh
        if odd == 1 and sh >= 1:
            kind, magic, sh = K_MAGIC, 1 << 63, sh - 1          # a / 2^sh = (a >> (sh-1)) / 2
        elif odd == 1:
            kind = K_SHIFT                                      # e == 1
        elif odd >> 32 == 0:
            kind, magic = K_MAGIC, M64 // odd + 1
        else:
            kind, sh = K_SLOW, 0
    dv = DimDiv(magic, e, sh, kind)
    if kind == K_SLOW:
        fast = False
    elif t < 2 and kind != K_MAGIC:
        fast = False
    elif kind != K_INF:
        fast = not (max_avail > 0 and (max_avail >> sh) >> 32 != 0)
    else:
        fast = True
    return dv, fast


def prep_fast32(fast: bool, c: DimDiv, m: DimDiv, shift32) -> bool:
    return (fast and c.kind == K_MAGIC and m.kind == K_MAGIC and c.sh >= shift32[0] and m.sh >= shift32[1]
            and c.sh - shift32[0] < 32 and m.sh - shift32[1] < 32)


def make_dimdiv(e: int) -> DimDiv:
    """The divider of reschedule / reschedule-from-reservations / reconcile: powers of two are plain shifts."""
    if e <= 0:
        return DimDiv(0, e, 0, K_INF)
    sh = ctz(e)
    odd = e >> sh
    if odd == 1:
        return DimDiv(0, e, sh, K_SHIFT)
    if odd >> 32 == 0:
        return DimDiv(M64 // odd + 1, e, sh, K_MAGIC)
    return DimDiv(0, e, 0, K_SLOW)


class SnapMeta:
    """Per-snapshot facts: largest availability per dimension (never below 0), the compact view's shifts, the
    negative-gpu flag."""

    def __init__(self, cpu, mem, gpu):
        self.max_avail = [max([0] + [int(x) for x in v]) for v in (cpu, mem, gpu)]
        self.shift32 = [shift_for(self.max_avail[0]), shift_for(self.max_avail[1])]
        self.gpu_negative = any(int(x) < 0 for x in gpu)


App = namedtuple("App", "drv exe count")


def prep_app(app: App, meta: SnapMeta):
    """-> (divs, fast, fast32) as gp_prep_apps computes them."""
    fast = True
    divs = []
    for t in range(3):
        dv, f = prep_dim(app.exe[t], t, meta.max_avail[t])
        divs.append(dv)
        fast = fast and f
    return divs, fast, prep_fast32(fast, divs[0], divs[1], meta.shift32)


def uses_gpu(app: App, meta: SnapMeta) -> bool:
    """The gpu dimension binds (kAppUsesGpu or kSnapGpuNegative): the hot path's gpu-idle specialisation is off."""
    return app.drv[2] != 0 or app.exe[2] != 0 or meta.gpu_negative


def classify(app: App, meta: SnapMeta):
    """-> (class pack_app dispatches to, (kind of cpu, mem, gpu)) for the independent scan."""
    divs, fast, f32 = prep_app(app, meta)
    idle = not uses_gpu(app, meta)
    cls = FAST32 if (f32 and idle) else FAST64 if (fast and idle) else GENERAL
    return cls, tuple(kind_name(d) for d in divs)


def family_class(family: str, app: App, meta: SnapMeta) -> str:
    """The arithmetic a kernel family uses for `app`: the scan dispatches three ways; minimal-fragmentation has
    MfCapFast32 and MfCapGeneral only; the FIFO kernels take FifoCaps<true> on kAppFast (gpu included) and never the
    compact view; the table build, the marker and the make_dimdiv users always divide with cap_dim."""
    divs, fast, f32 = prep_app(app, meta)
    idle = not uses_gpu(app, meta)
    if family == "scan":
        return classify(app, meta)[0]
    if family == "minfrag":
        return FAST32 if (f32 and idle) else GENERAL
    if family == "fifo":
        return FAST64 if fast else GENERAL
    return GENERAL


# ---- emulation of each class's arithmetic ----------------------------------------------------------------------------
def mulhi64(a: int, b: int) -> int:
    return ((a & M64) * (b & M64)) >> 64


def cap_dim_u(a: int, dv: DimDiv) -> int:
    """General class (cap_dim / cap_dim_u), unclamped; kDivInf -> None (unlimited)."""
    if a < 0:
        return 0
    if dv.kind == K_INF:
        return None
    xs = a >> dv.sh
    if dv.kind == K_SHIFT:
        return xs
    if dv.kind == K_MAGIC and xs >> 32 == 0:
        return mulhi64(dv.magic, xs)
    return a // dv.e                                            # udiv64


def _funnelshift_r(lo: int, hi: int, n: int) -> int:
    return ((((hi & M32) << 32) | (lo & M32)) >> (n & 31)) & M32


def fast_q(a: int, dv: DimDiv, magic_only: bool = False) -> int:
    """fast_q / fast_q_magic: a as two 32-bit words, a >> sh by one funnel shift, mulhi64(magic, xs) from a 32x32
    multiply plus one __umulhi; negative availability -> 0; kDivInf -> 0xFFFFFFFF."""
    u = a & M64
    lo, hi = u & M32, u >> 32
    big = dv.sh >= 32
    xs = _funnelshift_r(hi if big else lo, 0 if big else hi, dv.sh)
    m_lo, m_hi = dv.magic & M32, dv.magic >> 32
    q = ((m_hi * xs + ((m_lo * xs) >> 32)) >> 32) & M32
    if not magic_only:
        if dv.kind == K_SHIFT:
            q = xs
        if dv.kind == K_INF:
            q = M32
    return 0 if hi >> 31 else q


def compact_pair(v: int, s: int) -> int:
    return 0 if v < 0 else (v >> s) & M32


def cap32_dim(v32: int, dv: DimDiv, s: int) -> int:
    """Caps<true>::cap32 for one dimension: the compact value shifted by sh - S, then the 32-bit multiply-high."""
    xc = (v32 >> (dv.sh - s)) & M32
    m_lo, m_hi = dv.magic & M32, dv.magic >> 32
    return ((m_hi * xc + ((m_lo * xc) >> 32)) >> 32) & M32


def class_quotient(cls: str, a: int, dv: DimDiv, s: int = 0):
    """floor(a / e) the way class `cls` computes it (a is an availability minus a reservation; s the view's shift)."""
    if cls == GENERAL:
        return cap_dim_u(a, dv)
    if cls == FAST64:
        q = fast_q(a, dv, magic_only=False)
        return None if q == M32 and dv.kind == K_INF else q
    return cap32_dim(compact_pair(a, s), dv, s)


def exact_quotient(a: int, e: int):
    if a < 0:
        return 0
    return None if e == 0 else a // e


# ---- exact capacities, for choosing boundary counts ------------------------------------------------------------------
def node_cap(avail, reserved, exe):
    """min over dims of floor((avail - r) / e), None = unlimited."""
    out = None
    for d in range(3):
        a = avail[d] - reserved[d]
        q = exact_quotient(a, exe[d])
        if q is not None:
            out = q if out is None else min(out, q)
    return out
