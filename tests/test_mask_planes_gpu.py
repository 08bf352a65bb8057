"""The bit planes of the cron masks that the on-minute sweep reads (csrc/sweep_types.h, MaskPlanes): ticks that
together pick every plane, records flipping between UTC and zone-bound schedules inside one 32-record plane
word, and cron records at the word boundaries of a segment and in the last, partial tile of a shard — each
tick compared with the oracle."""
import numpy as np
import pytest

import oracle_c
from adversarial import ZoneMap, first_difference, zones_usable

pytestmark = pytest.mark.gpu

SEG = 128                 # records per segment: one warp of the sweep, 4 plane words
T_OCT = 1790812800        # 2026-10-01 00:00:00 UTC, Thursday
DAY, HOUR = 86400, 3600
FIELDS = {"minute": (0, 59), "hour": (0, 23), "dom": (1, 31), "month": (1, 12), "dow": (0, 6)}
STAR = np.uint64(1 << 63)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _field(rng, n, lo, hi):
    """masks of one field in every shape: a single value (the top one often), a range, a step, every value
    with the star bit, and a few with bits outside lo..hi that no tick can test"""
    bits = lambda vals: int(sum(1 << v for v in vals))
    out = np.empty(n, dtype=np.uint64)
    for i in range(n):
        shape = rng.integers(0, 6)
        if shape == 0:
            v = bits([int(rng.integers(lo, hi + 1))])
        elif shape == 1:
            v = bits([hi])
        elif shape == 2:
            a = int(rng.integers(lo, hi + 1))
            v = bits(range(a, int(rng.integers(a, hi + 1)) + 1))
        elif shape == 3:
            v = bits(range(int(rng.integers(lo, lo + 3)), hi + 1, int(rng.integers(2, 5))))
        elif shape == 4:
            v = bits(range(lo, hi + 1)) | (1 << 63)
        else:
            v = bits(v for v in range(lo, hi + 1) if rng.random() < 0.5)
        if rng.random() < 0.1:  # never tested: bit 0 of dom / month, bits past the field's top
            v |= bits([int(x) for x in rng.choice([b for b in range(63) if not lo <= b <= hi], 2)])
        out[i] = np.uint64(v)
    return out


def _columns(am, rng, n, T, cron):
    """n live records, `cron` (bool[n]) of them CRON_SPEC with masks of every shape; the others are
    interval-like kinds whose (also random) masks the sweep must ignore"""
    c = am.alloc_columns(n)
    for name, (lo, hi) in FIELDS.items():
        c[name][:] = _field(rng, n, lo, hi)
    # enough schedules that fire often: every minute / hour / month, the day rule then decides
    for name in ("minute", "hour", "month"):
        lo, hi = FIELDS[name]
        c[name][rng.random(n) < 0.4] = np.uint64(sum(1 << v for v in range(lo, hi + 1))) | STAR
    other = np.array([am.KIND_INTERVAL, am.KIND_CRON_EVERY, am.KIND_STOPPED, am.KIND_NO_RESOURCE,
                      am.KIND_PARSE_ERROR], dtype=np.uint32)
    kind = np.where(cron, np.uint32(am.KIND_CRON_SPEC), other[rng.integers(0, len(other), n)])
    c["flags"][:] = kind.astype(np.uint32) | np.uint32(am.F_TIMER_ARMED | am.F_STOPPED_REPORTED)
    c["ras"][:] = np.where(cron, 0, rng.integers(30, 150, n)).astype(np.int32)
    c["finished_at"][:] = T - rng.integers(0, 120, n)
    return c


def _tick_equal(am, s, ocols, T, sweep=oracle_c.sweep):
    got = s.tick(T)
    want = sweep(ocols, T)
    bad = first_difference(am, got, want, s.read_range(0, len(ocols["flags"])), ocols)
    assert bad is None, (T, bad)
    return len(want[0])


def _instants():
    """on-minute instants that together visit every minute of an hour, every hour of a day, every day of
    a 31-day month (seven consecutive weekdays among them) and the first of every month"""
    oct13 = T_OCT + 12 * DAY
    ts = [oct13 + 14 * HOUR + 60 * m for m in range(60)]
    ts += [oct13 + DAY + h * HOUR + 37 * 60 for h in range(24)]
    ts += [T_OCT + d * DAY + 5 * HOUR + 5 * 60 for d in range(31)]
    firsts = [1767225600, 1769904000, 1772323200, 1775001600, 1777593600, 1780272000,  # 2026-01-01 .. 06-01
              1782864000, 1785542400, 1788220800, T_OCT, 1793491200, 1796083200]       # 2026-07-01 .. 12-01
    ts += [t + 23 * HOUR + 59 * 60 for t in firsts]
    return ts


def test_ticks_that_pick_every_plane(am):
    """A few thousand records with masks of every shape (single values, ranges, steps, stars on dom and/or
    dow, dom 31, month 12, dow 6, stray bits no tick tests), ticked at instants that pick every minute,
    hour, day-of-month, month and weekday plane: each tick equals the oracle."""
    rng = np.random.default_rng(21)
    n = 3000
    ts = _instants()
    cols = _columns(am, rng, n, ts[0], rng.random(n) < 0.8)
    ocols = {k: v.copy() for k, v in cols.items()}
    fired = np.zeros(n, dtype=np.int64)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        for T in ts:
            got = s.tick(T)
            want = oracle_c.sweep(ocols, T)
            bad = first_difference(am, got, want, s.read_range(0, n), ocols)
            assert bad is None, (T, bad)
            fired[want[0].astype(np.int64)] += 1
    # many cron records fired at some ticks and not at others
    cron = (ocols["flags"] & np.uint32(7)) == am.KIND_CRON_SPEC
    assert ((fired > 0) & (fired < len(ts)) & cron).sum() > n // 4


@pytest.mark.parametrize("run", ["utc-to-zone", "zone-to-utc"])
def test_zone_binding_flips_within_one_plane_word(am, zmap, run):
    """Upserts inside one 32-record word turn UTC CRON_SPEC records into zone-bound ones and back.  A record
    that leaves UTC must lose its plane bits (its hour mask often names the UTC hour, rarely the zone's),
    and the zone path must pick it up; ticks at every hour of a day compared with the oracle."""
    rng = np.random.default_rng(22 if run == "utc-to-zone" else 23)
    n = 3 * 32 + 5
    T = T_OCT + 5 * DAY
    tz_ids = zmap.ids_of(zones_usable(T, T + 2 * DAY))
    assert tz_ids
    cols = _columns(am, rng, n, T, np.ones(n, dtype=bool))
    for name in ("minute", "month"):
        lo, hi = FIELDS[name]
        cols[name][:] = np.uint64(sum(1 << v for v in range(lo, hi + 1))) | STAR
    cols["dom"][:] = np.uint64(sum(1 << v for v in range(1, 32))) | STAR
    cols["dow"][:] = np.uint64(0x7F) | STAR
    cols["hour"][:] = rng.integers(0, 1 << 24, n, dtype=np.uint64)  # about half of the hours, per record
    word = np.arange(32, 64)
    zone = np.array(tz_ids, dtype=np.uint32)[rng.integers(0, len(tz_ids), n)]
    if run == "zone-to-utc":
        cols["flags"][word] |= zone[word] << np.uint32(24)
    ocols = {k: v.copy() for k, v in cols.items()}
    emitted = 0
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        for k in range(24):
            t = T + k * HOUR + 60 * int(rng.integers(0, 60))
            if k % 3 == 1:  # flip a third of the word's records: UTC <-> a zone
                idx = rng.choice(word, 11, replace=False)
                new = {name: ocols[name][idx].copy() for name in am.COLUMN_NAMES}
                bound = (new["flags"] >> np.uint32(24)) != 0
                new["flags"][:] = np.where(bound, new["flags"] & np.uint32(0x00FFFFFF),
                                           (new["flags"] & np.uint32(0x00FFFFFF)) | (zone[idx] << np.uint32(24)))
                new["hour"][:] = rng.integers(0, 1 << 24, len(idx), dtype=np.uint64)
                s.upsert(idx.astype(np.uint64), am.columns_to_records(new))
                for name in am.COLUMN_NAMES:
                    ocols[name][idx] = new[name]
            emitted += _tick_equal(am, s, ocols, t, sweep=zmap.sweep)
    assert emitted > 24 * n // 4


@pytest.mark.parametrize("path", ["load_range", "upsert"])
def test_cron_records_at_word_boundaries_and_in_a_partial_last_tile(am, path):
    """Cron records only at bits 0, 31, 32, 63, 64 and 127 of each segment (the first and last bit of each
    plane word a warp loads) in a shard of 2 * 1024 + 300 records, whose last tile is partial; ticks at
    several on-minute instants equal the oracle, and every one of those records fires at one of them."""
    rng = np.random.default_rng(24)
    n = 2 * 1024 + 300
    pos = np.array([0, 31, 32, 63, 64, 127])
    cron = np.zeros(n, dtype=bool)
    at = (np.arange(0, n, SEG)[:, None] + pos[None, :]).ravel()
    cron[at[at < n]] = True
    assert cron[2048:].sum() == 6 + 6 + 3  # segments 16, 17 and the partial 18 of the partial tile
    T = T_OCT + 12 * DAY + 14 * HOUR
    cols = _columns(am, rng, n, T, cron)
    ci = np.flatnonzero(cron)
    cols["minute"][ci] = np.uint64(1) << (ci % 8).astype(np.uint64)  # each fires at one of minutes 0..7
    for name in ("hour", "dom", "month", "dow"):
        lo, hi = FIELDS[name]
        cols[name][ci] = np.uint64(sum(1 << v for v in range(lo, hi + 1))) | STAR
    ocols = {k: v.copy() for k, v in cols.items()}
    fired = np.zeros(n, dtype=bool)
    with am.Sweep(capacity=n) as s:
        if path == "load_range":
            s.load_range(0, cols)
        else:
            order = rng.permutation(n).astype(np.uint64)
            s.upsert(order, am.columns_to_records({k: v[order.astype(np.int64)] for k, v in cols.items()}))
        for m in range(9):
            got = s.tick(T + 60 * m)
            want = oracle_c.sweep(ocols, T + 60 * m)
            assert first_difference(am, got, want, s.read_range(0, n), ocols) is None, m
            fired[want[0].astype(np.int64)] = True
    assert fired[ci].all()
