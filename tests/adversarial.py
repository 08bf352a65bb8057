"""The adversarial population of the sweep tests, shared by the CPU-emulator fuzz test
(tests/test_sweep_emulator_fuzz.py) and the device tests (tests/test_sweep_adversarial_gpu.py).

The values the generated BASELINE configs never reach — counters at INT32_MAX (wrap-around of
SuccessCount++ etc.), intervals of INT32_MAX, finishedAt exactly at / one second around the due
boundary or 2^40 away, remedy gates with limits and reset intervals at the i32 extremes, all-ones and
empty cron masks, armed and unarmed repeat timers, parse errors, "Stopped" reported and not yet
reported, the unsatisfiable schedule "0 0 30 2 *", schedules bound to named time zones — and, beyond
what the library itself can produce (`in_domain=False`), kinds 6/7, both PENDING bits at once, zero /
negative intervals on interval kinds and negative counters.

One combination is deliberately absent: AM_F_REMEDY_OUTCOME_OK without AM_F_REMEDY_PENDING.  It has no
meaning (post_result sets the two together); the oracle would clear the stray bit, the kernel leaves a
record with nothing pending untouched (include/amsweep.h, am_sweep_load_range).

Zone ids are handed out per registry (the product library, a second copy of it on the emulator, the C
oracle), in order of first appearance: `ZoneMap` translates the flags of one into the other's ids
around each oracle call, so columns are compared in the product's ids throughout."""
import ctypes as C
import importlib

import numpy as np

import amgen
import oracle_c

am = importlib.import_module("active-monitor_b200")
I32MIN, I32MAX = -(1 << 31), (1 << 31) - 1

# Instants: a Monday morning of 2026, the epoch and its neighbours, the i32 boundary, and far outside
# any calendar the controller will see.
TS = [1789982100, 1789982101, 0, -1, 59, 60, 1 << 31, -(1 << 33), (1 << 40) + 420, -(1 << 40), 1 << 54, -(1 << 54)]

# Africa/Monrovia kept local mean time, UTC-0:44:30, until 1972-01-07: an offset with seconds, which
# moves the local minute boundary off the UTC one.  The tz data of the period this project supports
# (1970 on) and both oracles agree on it; it is bound to records only at instants of 1970 and 1971.
MONROVIA = "Africa/Monrovia"
ZONE_NAMES = tuple(amgen.ZONES) + (MONROVIA,)
T_1972 = 63072000          # 1972-01-01 00:00:00 UTC
T_YEAR_10000 = 253402300800  # zone rules are compared with the oracles over years 1970 .. 9999 only


def zones_usable(T0, T1):
    """Names of the zones whose offsets the oracles are trusted with for every tick of [T0, T1]."""
    if T0 < 0 or T1 >= T_YEAR_10000:
        return []
    return list(amgen.ZONES) + ([MONROVIA] if T1 < T_1972 else [])


def product_lookup(lib=None):
    """zone name -> id in a build of the product library (default: the one `am` loads)"""
    lib = lib or am.load()

    def f(name):
        i = C.c_int32()
        assert lib.am_tz_lookup(name.encode(), len(name), C.byref(i)) == 0, name
        return i.value
    return f


def oracle_lookup(name):
    i = C.c_int32()
    assert oracle_c.load().orc_tz_lookup(name.encode(), len(name), C.byref(i)) == 0, name
    return i.value


class ZoneMap:
    """Zone ids of ZONE_NAMES in the product's registry and in the oracle's, both directions."""

    def __init__(self, lookup=None):
        lookup = lookup or product_lookup()
        self.ids = {z: lookup(z) for z in ZONE_NAMES}
        self.fwd = np.arange(256, dtype=np.uint32)
        self.back = np.arange(256, dtype=np.uint32)
        for z, p in self.ids.items():
            o = oracle_lookup(z)
            self.fwd[p] = o
            self.back[o] = p

    def ids_of(self, names):
        return [self.ids[z] for z in names]

    @staticmethod
    def _relabel(flags, lut):
        flags[:] = (flags & np.uint32(0x00FFFFFF)) | (lut[flags >> np.uint32(24)] << np.uint32(24))

    def sweep(self, ocols, T, **kw):
        """oracle_c.sweep on columns that carry the product's zone ids (in place, ids kept)"""
        self._relabel(ocols["flags"], self.fwd)
        try:
            return oracle_c.sweep(ocols, T, **kw)
        finally:
            self._relabel(ocols["flags"], self.back)


_FEB30 = None


def _feb30():
    global _FEB30
    if _FEB30 is None:
        _FEB30 = am.cron_parse("0 0 30 2 *")  # parses; never fires (robfig: Next() gives up)
    return _FEB30


def population(rng, n, T, in_domain=True, tz_ids=()):
    """SoA columns of `n` adversarial records around instant T.  `tz_ids`: zone ids (of the library the
    columns are loaded into) that 5-field schedules may be bound to — pick them with zones_usable()."""
    c = am.alloc_columns(n)
    for name in ("minute", "hour", "dom", "month", "dow"):
        v = rng.integers(0, 1 << 63, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
        sparse = rng.integers(0, 3, n) == 0
        v[sparse] = (np.uint64(1) << rng.integers(0, 62, n).astype(np.uint64))[sparse]
        v[rng.integers(0, 10, n) == 0] = 0
        v[rng.integers(0, 10, n) == 0] = np.uint64(0xFFFFFFFFFFFFFFFF)
        c[name][:] = v
    kind = rng.integers(0, 6 if in_domain else 8, n).astype(np.uint32)
    # the unsatisfiable schedule: a CRON_SPEC record that never fires
    feb = (kind == am.KIND_CRON_SPEC) & (rng.integers(0, 8, n) == 0)
    fc = _feb30()
    for name in ("minute", "hour", "dom", "month", "dow"):
        c[name][feb] = np.uint64(getattr(fc, name))
    flags = kind.copy()
    flags |= (rng.integers(0, 2, n).astype(np.uint32) << 3)          # HAS_REMEDY
    ph = rng.integers(0, 3 if in_domain else 4, n)                   # none / ok / fail / (both)
    flags |= np.where(ph == 1, am.F_PENDING_OK, 0).astype(np.uint32)
    flags |= np.where(ph == 2, am.F_PENDING_FAIL, 0).astype(np.uint32)
    flags |= np.where(ph == 3, am.F_PENDING_OK | am.F_PENDING_FAIL, 0).astype(np.uint32)
    rp = rng.integers(0, 3, n)
    flags |= np.where(rp == 1, am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK, 0).astype(np.uint32)
    flags |= np.where(rp == 2, am.F_REMEDY_PENDING, 0).astype(np.uint32)
    flags |= np.where(rng.integers(0, 20, n) == 0, am.F_TOMBSTONE, 0).astype(np.uint32)
    flags |= np.where(rng.integers(0, 4, n) == 0, am.F_STOPPED_REPORTED, 0).astype(np.uint32)
    flags |= np.where(rng.integers(0, 2, n) == 0, am.F_TIMER_ARMED, 0).astype(np.uint32)
    flags |= (rng.integers(0, 256, n).astype(np.uint32) << 16)       # closed-loop P(fail)
    if len(tz_ids):
        bound = (kind == am.KIND_CRON_SPEC) & (rng.integers(0, 3, n) != 0)
        zone = np.array(tz_ids, dtype=np.uint32)[rng.integers(0, len(tz_ids), n)]
        flags |= np.where(bound, zone << np.uint32(24), 0).astype(np.uint32)
    c["flags"][:] = flags
    pick = lambda opts: np.array(opts, dtype=np.int64)[rng.integers(0, len(opts), n)]
    ras = pick([1, 5, 60, 3600, I32MAX, 7, 86400] + ([] if in_domain else [0, -1, I32MIN]))
    c["ras"][:] = ras.astype(np.int32)
    fa_rel = pick([0, 1, -1, 59, 60, 61, 3600, 100000])
    fa = T - ras + fa_rel
    alt = pick([0, T, T + 1, T - 1, T + 100, -(1 << 40), (1 << 40)])
    use_alt = rng.integers(0, 3, n) == 0
    fa = np.where(use_alt, alt, fa)
    c["finished_at"][:] = fa
    c["runs_limit"][:] = pick([0, 1, 2, 5, -1, I32MAX, I32MIN]).astype(np.int32)
    c["reset_interval"][:] = pick([0, 60, 300, -1, 1, I32MAX, I32MIN]).astype(np.int32)
    for name in ("success", "failed"):
        c[name][:] = pick([0, 1, 7, 1000, I32MAX, I32MAX - 1] + ([] if in_domain else [-1, I32MIN])).astype(np.int32)
    rs = pick([0, 1, 2, 3, I32MAX] + ([] if in_domain else [-1])).astype(np.int64)
    rf = pick([0, 1, 2, 3, I32MAX] + ([] if in_domain else [-5])).astype(np.int64)
    c["remedy_success"][:] = rs.astype(np.int32)
    c["remedy_failed"][:] = rf.astype(np.int32)
    rt = np.where(rng.integers(0, 4, n) == 0, pick([0, 1, 2, 6, -1, I32MAX]), rs + rf)
    c["remedy_total"][:] = (rt & 0xFFFFFFFF).astype(np.uint32).view(np.int32)
    rst = c["reset_interval"].astype(np.int64)
    rfa = T - rst + pick([0, 1, -1, 5])
    rfa = np.where(rng.integers(0, 3, n) == 0, pick([0, 0, T, T + 5, -(1 << 40), (1 << 40), T - (1 << 34), T + (1 << 34)]), rfa)
    c["remedy_finished_at"][:] = rfa
    return c


def first_difference(am_, got, want, dev, ocols):
    """None when a tick's (list, actions, statistics) and the columns after it equal the oracle's;
    else a description of the first difference"""
    gi, ga, gs = got
    wi, wa, ws = want
    if gs != ws:
        return ("stats", {f: (gs[f], ws[f]) for f in gs if gs[f] != ws[f]})
    if not np.array_equal(gi, wi):
        return ("idx",)
    if not np.array_equal(ga, wa):
        return ("act",)
    for name in am_.COLUMN_NAMES:
        if not np.array_equal(dev[name], ocols[name]):
            i = int(np.flatnonzero(dev[name] != ocols[name])[0])
            return ("col", name, i, int(dev[name][i]), int(ocols[name][i]))
    return None


def run_single_ticks(make_sweep, zmap, seed, n, T, mode, in_domain, ticks=3):
    """`ticks` consecutive host ticks of an adversarial population from T on, each compared with the
    oracle; None, or (seed, n, T, mode, tick, difference)."""
    rng = np.random.default_rng(seed)
    cols = population(rng, n, T, in_domain, zmap.ids_of(zones_usable(T, T + ticks)))
    ocols = {k: v.copy() for k, v in cols.items()}
    with make_sweep(n) as s:
        s.load_range(0, cols)
        s.set_seed(seed)
        for k in range(ticks):
            got = s.tick(T + k, mode=mode)
            want = zmap.sweep(ocols, T + k, mode=mode & 1, seed=seed)
            bad = first_difference(am, got, want, s.read_range(0, n), ocols)
            if bad:
                return (seed, n, T, mode, k, bad)
    return None
