"""The packed copy of the cron masks that the on-minute sweep reads (csrc/sweep_types.h, PackedMasks): every
way the library writes masks or kind bits — bulk loads at ragged offsets, upserts and removes that flip
records between CRON_SPEC and other kinds, drains done by a read, next-due or repeat-after query — followed
by on-minute ticks compared with the oracle, at per-segment cron counts from 0 to 128 and with schedules
bound to named time zones.  Every schedule is different, so a stale or shifted pack changes the due set."""
import numpy as np
import pytest

import oracle_c
from adversarial import ZoneMap, first_difference, population, zones_usable

pytestmark = pytest.mark.gpu

SEG = 128                 # records per segment: one warp of the sweep
T0 = 1789982100           # 2026-09-21 09:15:00 UTC Monday, on the minute
T_LORD_HOWE = 1790004600  # 2026-09-21 15:30:00 UTC: 02:00 in Lord Howe (+10:30)
T_MONROVIA = 44618400     # 1971-06-01 10:00:00 UTC: Monrovia's clock reads 09:15:30 (UTC-0:44:30)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _masks(rng, n):
    """distinct schedules: random minutes and hours, every day of every month"""
    out = {
        "minute": rng.integers(0, 1 << 60, n, dtype=np.uint64),
        "hour": rng.integers(0, 1 << 24, n, dtype=np.uint64) | np.uint64(1 << 9) | np.uint64(1 << 15),
        "dom": np.full(n, ((1 << 32) - 2) | (1 << 63), dtype=np.uint64),
        "month": np.full(n, ((1 << 13) - 2) | (1 << 63), dtype=np.uint64),
        "dow": np.full(n, ((1 << 7) - 1) | (1 << 63), dtype=np.uint64),
    }
    return out


def _records(am, rng, n, T, cron):
    """columns of n live records; `cron` (bool[n]) picks CRON_SPEC, the others get one of the other kinds.
    Every record carries masks of its own, the non-cron ones too (the library must ignore those)."""
    c = am.alloc_columns(n)
    for name, v in _masks(rng, n).items():
        c[name][:] = v
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


def _upsert(s, ocols, idx, recs_cols, am):
    recs = am.columns_to_records(recs_cols)
    s.upsert(idx, recs)
    for name in am.COLUMN_NAMES:
        ocols[name][idx] = recs_cols[name]
    ocols["flags"][idx] &= ~np.uint32(am.F_TOMBSTONE)


def _remove(s, ocols, idx, am):
    s.remove(idx)
    ocols["flags"][idx] = np.uint32(am.F_TOMBSTONE)


def _is_cron(am, cols):
    return (cols["flags"] & np.uint32(7)) == am.KIND_CRON_SPEC


def test_upserts_and_removes_flip_kinds_within_a_segment(am):
    """Batches of upserts and removes confined to one segment turn CRON_SPEC records into other kinds and
    back (and remove cron records outright, which shifts every later slot of the segment); an on-minute
    tick after each batch equals the oracle."""
    rng = np.random.default_rng(11)
    n = 3 * SEG
    cols = _records(am, rng, n, T0, rng.random(n) < 0.5)
    ocols = {k: v.copy() for k, v in cols.items()}
    emitted = 0
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        emitted += _tick_equal(am, s, ocols, T0)
        for b in range(12):
            T = T0 + 60 * (b + 1)
            seg = 1 + (b % 2)
            idx = (seg * SEG + rng.choice(SEG, 24, replace=False)).astype(np.uint64)
            if b % 3 == 2:  # removes only: some cron records of the segment disappear
                crons = idx[_is_cron(am, ocols)[idx.astype(np.int64)]]
                _remove(s, ocols, crons[: max(1, len(crons) // 2)], am)
            else:  # flip the kind of every chosen record, with new schedules
                flip = ~_is_cron(am, ocols)[idx.astype(np.int64)]
                _upsert(s, ocols, idx, _records(am, rng, len(idx), T, flip), am)
                if b % 3 == 1:  # ... and remove a few other cron records of the segment in the same drain
                    rest = np.setdiff1d(np.arange(seg * SEG, (seg + 1) * SEG), idx.astype(np.int64))
                    _remove(s, ocols, rest[_is_cron(am, ocols)[rest]][:3].astype(np.uint64), am)
            emitted += _tick_equal(am, s, ocols, T)
    assert emitted > 100


@pytest.mark.parametrize("path", ["load_range", "upsert"])
def test_segments_with_0_1_63_64_65_128_cron_records(am, path):
    """Six segments holding 0, 1, 63, 64, 65 and 128 cron records at random positions (the packed slots
    fill no, one, part of, exactly one, just over one and both halves of a warp's loads), loaded in bulk or
    upserted into a fresh handle; five on-minute ticks equal the oracle."""
    rng = np.random.default_rng(12)
    counts = [0, 1, 63, 64, 65, 128]
    n = SEG * len(counts)
    cron = np.zeros(n, dtype=bool)
    for k, c in enumerate(counts):
        cron[k * SEG + rng.choice(SEG, c, replace=False)] = True
    cols = _records(am, rng, n, T0, cron)
    ocols = {k: v.copy() for k, v in cols.items()}
    emitted = 0
    with am.Sweep(capacity=n) as s:
        if path == "load_range":
            s.load_range(0, cols)
        else:
            order = rng.permutation(n).astype(np.uint64)
            s.upsert(order, am.columns_to_records({k: v[order.astype(np.int64)] for k, v in cols.items()}))
        for k in range(5):
            emitted += _tick_equal(am, s, ocols, T0 + 60 * k)
    assert emitted > 200


def test_load_range_at_ragged_offsets_over_existing_data(am):
    """am_sweep_load_range over data already loaded, at offsets and lengths that are not multiples of the
    segment: partial segments at both ends of a range, ranges spanning several segments, a single record."""
    rng = np.random.default_rng(13)
    n = 1000
    cols = _records(am, rng, n, T0, rng.random(n) < 0.4)
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        _tick_equal(am, s, ocols, T0)
        for k, (first, m) in enumerate([(37, 300), (500, 129), (700, 1), (127, 2), (255, 514), (999, 1), (0, 1000)]):
            T = T0 + 60 * (k + 1)
            part = _records(am, rng, m, T, rng.random(m) < (0.9 if k % 2 else 0.1))
            s.load_range(first, part)
            for name in am.COLUMN_NAMES:
                ocols[name][first:first + m] = part[name]
            assert _tick_equal(am, s, ocols, T) > 0


@pytest.mark.parametrize("drain", ["read", "read_idx", "next_due", "repeat_after"])
def test_a_drain_by_a_query_then_a_tick(am, drain):
    """Upserts and removes drained by a read, a next-due or a repeat-after query (not by a tick): the next
    on-minute tick sees them."""
    rng = np.random.default_rng(14)
    n = 2 * SEG + 17
    cols = _records(am, rng, n, T0, rng.random(n) < 0.5)
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        for b in range(4):
            T = T0 + 60 * b
            idx = rng.choice(n, 30, replace=False).astype(np.uint64)
            flip = ~_is_cron(am, ocols)[idx.astype(np.int64)]
            _upsert(s, ocols, idx, _records(am, rng, len(idx), T, flip), am)
            rest = np.setdiff1d(np.arange(n), idx.astype(np.int64))
            gone = rest[_is_cron(am, ocols)[rest]][:4].astype(np.uint64)
            _remove(s, ocols, gone, am)
            if drain == "read":
                s.read_range(0, n)
            elif drain == "read_idx":
                s.read(idx[:5])
            elif drain == "next_due":
                s.next_due(T - 1)
            else:
                s.repeat_after_sec(T - 1, 0, n)
            _tick_equal(am, s, ocols, T)


ZONE_RUNS = [("lord-howe", T_LORD_HOWE, 6), ("monrovia", T_MONROVIA, 4), ("2026", T0, 4)]


@pytest.mark.parametrize("run_id,T,nt", ZONE_RUNS, ids=[r[0] for r in ZONE_RUNS])
def test_zone_bound_schedules_in_packed_slots(am, zmap, run_id, T, nt):
    """Schedules bound to named time zones (their id travels with the packed hour word) among UTC ones, at
    cron densities that fill different numbers of slots; every tick of a few minutes (in 1971 Monrovia's
    offset has seconds, so every second reads the masks) and upserts flipping zone-bound records."""
    rng = np.random.default_rng(15 + len(run_id))
    n = 4 * SEG + 9
    tz_ids = zmap.ids_of(zones_usable(T, T + 60 * nt))
    assert tz_ids
    cols = population(rng, n, T, True, tz_ids)
    fl = cols["flags"]
    dense = (np.arange(n) // SEG) % 2 == 1  # every other segment mostly cron, zone-bound or not
    make_cron = dense & (rng.random(n) < 0.85)
    fl[:] = np.where(make_cron, (fl & ~np.uint32(7)) | am.KIND_CRON_SPEC, fl)
    zone = np.array(tz_ids, dtype=np.uint32)[rng.integers(0, len(tz_ids), n)]
    bind = make_cron & (rng.random(n) < 0.5)
    fl[:] = np.where(bind, (fl & np.uint32(0x00FFFFFF)) | (zone << np.uint32(24)), fl)
    star = rng.random(n) < 0.5  # fire somewhere in every zone's minute
    cols["minute"][star] = np.uint64((1 << 60) - 1)
    cols["hour"][star] = np.uint64((1 << 24) - 1)
    cols["dom"][star] = np.uint64(((1 << 32) - 2) | (1 << 63))
    cols["month"][star] = np.uint64(((1 << 13) - 2) | (1 << 63))
    cols["dow"][star] = np.uint64(((1 << 7) - 1) | (1 << 63))
    ocols = {k: v.copy() for k, v in cols.items()}
    emitted = 0
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        for k in range(nt * 60 if run_id == "monrovia" else nt):
            t = T + (k if run_id == "monrovia" else 60 * k)
            if k % 7 == 3:  # flip a few records of a dense segment between zone-bound cron and other kinds
                idx = (SEG + rng.choice(SEG, 12, replace=False)).astype(np.uint64)
                new = population(rng, len(idx), t, True, tz_ids)
                is_c = _is_cron(am, ocols)[idx.astype(np.int64)]
                nf = new["flags"]
                nf[:] = np.where(is_c, (nf & ~np.uint32(7)) | am.KIND_INTERVAL,
                                 (nf & np.uint32(0x00FFFFF8)) | am.KIND_CRON_SPEC | (zone[: len(idx)] << np.uint32(24)))
                _upsert(s, ocols, idx, new, am)
            emitted += _tick_equal(am, s, ocols, t, sweep=zmap.sweep)
    assert emitted > 50
