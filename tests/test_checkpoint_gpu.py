"""am_sweep_checkpoint / am_sweep_restore: a restore is the identity on the handle model (tests/handle_model.py), so a
walk checkpoints the pair's handle, restores into fresh handles, points the pair at the restored one and goes on
comparing with the unchanged model.  Random call sequences on the adversarial population (zones, timeouts, remedies)
under every switch combination, with and without the timeout state, restores with calls staged on both sides, into a
larger capacity and as two blobs in reverse order, then a catch-up tick across a gap; a simulated run split by a
restart; resharding one handle into two and three; a blob restored in a process whose zone registry has another
order; every refusal; the numpy reader of the format (tests/checkpoint_format.py); and 10 M records."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest

import checkpoint_format as fmt
from adversarial import ZONE_NAMES, ZoneMap, population, zones_usable
from handle_pair import Pair, emulated

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DAY = 86400
CATCH, BLOCKED = 0x8, 0x4
T_PARIS = 1792890000 - 400  # Europe/Paris leaves summer time at 1792890000 (2026-10-25 01:00 UTC)
T_OCT = 1790812800 + 37
SWITCHES = {"off": {}, "hold": dict(hold=True), "hold_remedy": dict(hold=True, remedy=True),
            "track": dict(track=True), "track_details": dict(track=True, details=True)}


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _records(am, zmap, rng, n, T, timeouts):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
    recs["wf_timeout"] = np.where(rng.random(n) < 0.4, 0, rng.integers(1, 40, n)) if timeouts else 0
    return recs


def _fresh(am, capacity, shard_base, info):
    """a handle with a blob's switches, set as a controller sets them after am_checkpoint_info"""
    s = am.Sweep(capacity=capacity, shard_base=shard_base)
    sw = info["switches"]
    if sw & am.CKPT_HOLD:
        s.set_hold_in_flight(True)
    if sw & am.CKPT_REMEDY:
        s.set_hold_remedy(True)
    if sw & am.CKPT_TRACK:
        s.set_track_changes(True)
    if sw & am.CKPT_DETAILS:
        s.set_change_details(True)
    return s


def _same_answers(am, a, b, n, T, where):
    """the queries of the equivalence, handle against handle, over the first n slots"""
    ga, gb = a.read_range(0, n), b.read_range(0, n)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(gb[name], ga[name], err_msg=f"{where}: {name}")
    for fn in ("in_flight", "remedy_in_flight"):
        np.testing.assert_array_equal(getattr(b, fn)(0, n), getattr(a, fn)(0, n), err_msg=f"{where}: {fn}")
    np.testing.assert_array_equal(b.repeat_after_sec(T, 0, n), a.repeat_after_sec(T, 0, n), err_msg=f"{where}: ras")
    assert b.next_due(T) == a.next_due(T), where


def _check_format(am, p, blob, first, n):
    """the numpy reader's sections equal what the source answers"""
    r = fmt.read(blob)
    assert r["checksum_ok"] and r["first_global"] == p.s.shard_base + first and r["n"] == n
    cols = p.s.read_range(first, n)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(r[name], cols[name], err_msg=name)
    if p.m.hold:
        since = r["since"]
        hc = np.where(since >= (1 << 59), np.int64(-(1 << 63)), since)
        inf = p.s.in_flight(first, n)
        held = inf != -(1 << 63)
        np.testing.assert_array_equal(hc[held], inf[held])  # (a since the next tick ignores reads as not in flight)
        if p.m.remedy:
            rinf = p.s.remedy_in_flight(first, n)
            rh = rinf != -(1 << 63)
            np.testing.assert_array_equal(since[rh] - (1 << 60), rinf[rh])
    info = am.checkpoint_info(blob)
    for k in ("first_global", "n", "swept_end", "seed", "n_zones", "bytes", "switches"):
        assert info[k] == r[k], k
    return r


def _restore(am, p, blobs, capacity=None, stage_target=False, rng=None, T=None):
    """restore `blobs` (in the given order) into a fresh handle of the pair's shard, optionally with calls staged on it
    that the restore replaces; check the queries against the source; the pair goes on with the restored handle"""
    info = am.checkpoint_info(blobs[0])
    t = _fresh(am, capacity or p.n, p.s.shard_base, info)
    if stage_target:
        sl = rng.choice(p.m.hwm, 7, replace=False)  # (a drained upsert raises the high-water mark)
        t.upsert(sl, _junk(am, len(sl)))
        t.post_result(sl[:4], np.array([1, 2, 1, 2], np.uint8), np.array([0, 1, 2, 0], np.uint8))
    for b in blobs:
        t.restore(b)
    _same_answers(am, p.s, t, p.n, T, "restore")
    p.s.close()
    p.s = t


def _junk(am, k):
    rc, r = am.classify(repeat_after_sec=1, finished_at=0)
    assert rc == 0
    return np.repeat(r, k)


def _random_call(am, zmap, p, rng, T, timeouts):
    n = p.n
    c = rng.integers(0, 6)
    if c == 0:
        sl = rng.choice(n, rng.integers(1, 40), replace=True)
        p.upsert(sl, _records(am, zmap, rng, len(sl), T, timeouts))
    elif c == 1:
        p.remove(rng.choice(n, rng.integers(1, 10), replace=False))
    elif c in (2, 3):
        sl = rng.choice(p.m.hwm, rng.integers(1, 80), replace=True)  # (posts go to swept slots)
        p.post(sl, rng.integers(0, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8))
    else:
        p.read(rng.choice(n, 5))


@pytest.mark.parametrize("timeouts", [False, True], ids=["no_timeouts", "timeouts"])
@pytest.mark.parametrize("switches", list(SWITCHES))
def test_walk(am, zmap, switches, timeouts):
    rng = np.random.default_rng(zlib.crc32(f"{switches} {timeouts}".encode()))
    n = 700
    T = T_PARIS
    p = Pair(am, zmap, n, seed=11, every_slot=False, **SWITCHES[switches])  # (removes leave stale columns)
    try:
        p.upsert(np.arange(n - 37), _records(am, zmap, rng, n - 37, T, timeouts))  # (the last slots never swept)
        restores = {6: "staged", 13: "larger", 20: "two_blobs_reversed", 27: "staged"}
        for step in range(34):
            for _ in range(rng.integers(0, 3)):
                _random_call(am, zmap, p, rng, T, timeouts)
            kind = restores.get(step)
            if kind:
                p.post(rng.choice(p.m.hwm, 9), np.full(9, 2, np.uint8))  # (staged on the source: the checkpoint drains it)
                p.upsert(rng.choice(n, 3), _records(am, zmap, rng, 3, T, timeouts))
                if kind == "two_blobs_reversed":
                    a = int(rng.integers(1, n))
                    blobs = [p.s.checkpoint(a, n - a), p.s.checkpoint(0, a)]
                    _check_format(am, p, blobs[0], a, n - a)
                else:
                    blobs = [p.s.checkpoint(0, n)]
                    _check_format(am, p, blobs[0], 0, n)
                _restore(am, p, blobs, capacity=n + 1500 if kind == "larger" else None, stage_target=kind == "staged",
                         rng=rng, T=T)
            T += int(rng.choice([1, 1, 2, 7, 30, 60]))
            p.tick(T, mode=CATCH if rng.random() < 0.3 else 0)
        # a restart across a gap: restore, then one catch-up tick 15 minutes later
        blob = p.s.checkpoint(0, n)
        _restore(am, p, [blob], T=T)
        T += 900
        before = p.timed_total + p.rtimed_total
        assert p.m.window_of(T, CATCH) == T - 900  # (the model's P: the handle must have it from the blob)
        got = p.tick(T, mode=CATCH)
        assert got.stats["n_submit_hc"] > 0 or p.m.hold, got.stats
        if p.m.hold and timeouts:
            assert p.timed_total + p.rtimed_total > before, "expired deadlines time out at the first tick"
        for k in range(1, 4):
            p.tick(T + k)
    finally:
        p.close()


def _sim_handle(am, zmap, recs, n, T0, rng_posts):
    s = am.Sweep(capacity=n)
    s.set_hold_in_flight(True)
    s.set_hold_remedy(True)
    s.upsert(np.arange(n), recs)
    for T in (T0 - 6, T0 - 2):
        s.tick(T)
    sl, ph, rp = rng_posts
    s.post_result(sl, ph, rp)
    return s


@pytest.mark.parametrize("mode", [0, BLOCKED], ids=["ticks", "blocked"])
def test_simulated_day_split_by_a_restart(am, zmap, mode):
    rng = np.random.default_rng(5 + mode)
    n, K = 512, 300
    recs = _records(am, zmap, rng, n, T_OCT, True)
    recs["wf_timeout"] = np.where(rng.random(n) < 0.5, 0, rng.integers(1, 6, n))
    sl = rng.choice(n, n // 10, replace=False)
    posts = (sl, rng.integers(0, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8))
    params = (1, 5, 1, 4)
    whole = _sim_handle(am, zmap, recs, n, T_OCT, posts)
    half = _sim_handle(am, zmap, recs, n, T_OCT, posts)
    try:
        rows, sims = whole.simulate(T_OCT, K, mode, 3, params)
        r1, s1 = half.simulate(T_OCT, K // 2, mode, 3, params)
        blob = half.checkpoint(0, n)
        half.close()
        half = _fresh(am, n, 0, am.checkpoint_info(blob))
        half.restore(blob)
        r2, s2 = half.simulate(T_OCT + K // 2, K - K // 2, mode, 3, params)
        np.testing.assert_array_equal(np.concatenate([r1, r2]), rows)
        np.testing.assert_array_equal(np.concatenate([s1, s2]), sims)
        assert sims["n_in_flight"].max() > 0 and sims["n_timed_out"].sum() > 0
        _same_answers(am, whole, half, n, T_OCT + K, "after the simulation")
    finally:
        whole.close()
        half.close()


def _sum_stats(stats):
    out = {k: sum(s[k] for s in stats) for k in stats[0] if k not in ("n_records", "idx_xor")}
    x = 0
    for s in stats:
        x ^= s["idx_xor"]
    out["idx_xor"] = x
    return out


@pytest.mark.parametrize("layout", ["two", "three"])
def test_resharding(am, zmap, layout):
    """one handle's checkpoint restored into two or three shards (other bases and capacities, one GPU): the
    concatenated lists, the summed statistics, the timed-out lists and the columns follow the model"""
    rng = np.random.default_rng(len(layout))
    n = 900
    T = T_PARIS
    p = Pair(am, zmap, n, hold=True, remedy=True, track=True)
    shards = []
    try:
        p.upsert(np.arange(n), _records(am, zmap, rng, n, T, True))
        for k in range(6):
            T += 7
            p.tick(T)
            _random_call(am, zmap, p, rng, T, True)
        cuts = [0, 333, n] if layout == "two" else [0, 211, 640, n]
        blobs = [p.s.checkpoint(a, b - a) for a, b in zip(cuts, cuts[1:])]
        # shard k holds [cuts[k], cuts[k+1]); the middle one's base is below its first slot, its capacity larger
        for k, blob in enumerate(blobs):
            base = cuts[k] - (5 if k == 1 else 0)
            s = _fresh(am, cuts[k + 1] - base + 100 * k, base, am.checkpoint_info(blob))
            s.restore(blob)
            shards.append(s)
        for step in range(40):
            T += int(rng.choice([1, 3, 20, 60]))
            if step % 3 == 0:
                sl = rng.choice(n, 30)
                ph, rp = rng.integers(0, 3, 30).astype(np.uint8), rng.integers(0, 3, 30).astype(np.uint8)
                p.m.post(sl, ph, rp)
                for k, s in enumerate(shards):
                    m = (sl >= cuts[k]) & (sl < cuts[k + 1])
                    if m.any():
                        s.post_result(sl[m] - s.shard_base, ph[m], rp[m])
            want = p.m.tick(T, 0)
            got = [s.tick(T) for s in shards]
            np.testing.assert_array_equal(np.concatenate([g[0] for g in got]), want.idx, err_msg=str(T))
            np.testing.assert_array_equal(np.concatenate([g[1] for g in got]), want.act, err_msg=str(T))
            ws = dict(want.stats)
            ws.pop("n_records")
            assert _sum_stats([g[2] for g in got]) == ws, T
            for k in range(2):
                np.testing.assert_array_equal(np.concatenate([s.last_timed_out()[k] for s in shards]), want.timed_out[k])
                np.testing.assert_array_equal(np.concatenate([s.last_remedy_timed_out()[k] for s in shards]),
                                              want.remedy_timed_out[k])
            np.testing.assert_array_equal(np.concatenate([s.last_changes()[0] for s in shards]), p.m.changes())
        mc = p.m.cols()
        for k, s in enumerate(shards):
            lo = cuts[k] - s.shard_base
            got = s.read_range(lo, cuts[k + 1] - cuts[k])
            live = p.m.live(np.arange(cuts[k], cuts[k + 1]))  # (removes leave stale columns)
            for name in am.COLUMN_NAMES:
                keep = live | (name == "flags")
                np.testing.assert_array_equal(got[name][keep], mc[name][cuts[k]:cuts[k + 1]][keep], err_msg=name)
    finally:
        for s in shards:
            s.close()
        p.close()


CHILD = r"""
import ctypes as C, importlib, json, sys
import numpy as np
sys.path.insert(0, {root!r})
am = importlib.import_module("active-monitor_b200")
names = {names!r}
ids = {{z: am.tz_lookup(z) for z in names}}  # another order than the parent's
blob = open({path!r}, "rb").read()
info = am.checkpoint_info(blob)
s = am.Sweep(capacity=info["n"])
s.set_hold_in_flight(True)
s.restore(blob)
out = {{"ids": ids, "ticks": []}}
for T in {ticks!r}:
    i, a, st = s.tick(T, mode=8)
    out["ticks"].append([i.tolist(), a.tolist(), st])
cols = s.read_range(0, info["n"])
out["cols"] = {{k: v.tolist() for k, v in cols.items()}}
out["in_flight"] = s.in_flight(0, info["n"]).tolist()
print(json.dumps(out))
"""


def test_another_zone_registry(am, zmap):
    """a blob restored in a child process that registered the zones in reverse order ticks across a daylight-saving
    transition exactly as the original"""
    rng = np.random.default_rng(9)
    n = 600
    T = 1792890000 - 181  # Europe/Paris and its neighbours leave summer time at 1792890000
    s = am.Sweep(capacity=n)
    s.set_hold_in_flight(True)
    try:
        recs = _records(am, zmap, rng, n, T, True)
        s.upsert(np.arange(n), recs)
        s.tick(T)
        ticks = [T + 60 * k + 1 for k in range(1, 9)]
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "blob")
            with open(path, "wb") as f:
                f.write(s.checkpoint(0, n))
            code = CHILD.format(root=ROOT, names=list(reversed(ZONE_NAMES)), path=path, ticks=ticks)
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        child = json.loads(r.stdout.strip().splitlines()[-1])
        lut = np.zeros(256, np.uint32)  # the child's id -> this process's id
        for z, i in child["ids"].items():
            lut[i] = zmap.ids[z]
        assert any(child["ids"][z] != zmap.ids[z] for z in child["ids"])
        for T, (ci, ca, cs) in zip(ticks, child["ticks"]):
            i, a, st = s.tick(T, mode=CATCH)
            assert ci == i.tolist() and ca == a.tolist() and cs == st, T
        cols = s.read_range(0, n)
        f = np.array(child["cols"]["flags"], np.uint32)
        bound = (f & np.uint32(7)) == am.KIND_CRON_SPEC
        f[bound] = (f[bound] & np.uint32(0xFFFFFF)) | (lut[f[bound] >> np.uint32(24)] << np.uint32(24))
        np.testing.assert_array_equal(f, cols["flags"])
        for name in am.COLUMN_NAMES:
            if name != "flags":
                np.testing.assert_array_equal(np.array(child["cols"][name], dtype=cols[name].dtype), cols[name], name)
        np.testing.assert_array_equal(child["in_flight"], s.in_flight(0, n))
    finally:
        s.close()


def _edit(blob, at, value, size=8):
    b = bytearray(blob)
    b[at:at + size] = int(value).to_bytes(size, "little", signed=value < 0)
    return fmt.reseal(bytes(b))


def test_refusals_change_nothing(am, zmap):
    """every refusal leaves the target as it was: a read and a tick equal a control handle's"""
    rng = np.random.default_rng(4)
    n = 300
    T = T_PARIS
    src = am.Sweep(capacity=n)
    src.set_hold_in_flight(True)
    recs = _records(am, zmap, rng, n, T, True)
    src.upsert(np.arange(n), recs)
    src.tick(T)
    blob = src.checkpoint(0, n)
    src.close()
    info = am.checkpoint_info(blob)
    assert info["n_zones"] > 0 and info["prev_tick"] == T and info["switches"] == am.CKPT_HOLD | am.CKPT_TIMEOUTS
    r = fmt.read(blob)
    zid, zname = next(iter(r["zones"].items()))
    end = fmt.sections(n, int(info["switches"]))[1]
    name_at = end + 8
    bad_zone = bytearray(blob)
    bad_zone[name_at:name_at + len(zname)] = b"X" * len(zname)
    version_at = fmt.HEADER_FIELDS.fields["version"][1]
    flip = bytearray(blob)
    flip[200] ^= 1
    cases = [
        ("truncated", blob[:-8], {}, am.AM_E_INVAL),
        ("bad checksum", bytes(flip), {}, am.AM_E_INVAL),
        ("version", _edit(blob, version_at, 2, 4), {}, am.AM_E_INVAL),
        ("switches", blob, dict(hold=False), am.AM_E_INVAL),
        ("previous tick", blob, dict(P=T - 1), am.AM_E_INVAL),
        ("unknown zone", fmt.reseal(bytes(bad_zone)), {}, am.AM_E_PARSE),
        ("base past the first slot", blob, dict(base=1), am.AM_E_RANGE),
        ("capacity", blob, dict(capacity=n - 1), am.AM_E_RANGE),
    ]
    for what, b, kw, code in cases:
        pair, probe = [], []
        for _ in range(2):  # the target, and its control
            s = am.Sweep(capacity=kw.get("capacity", n), shard_base=kw.get("base", 0))
            if kw.get("hold", True):
                s.set_hold_in_flight(True)
            s.upsert([3], _junk(am, 1))
            if "P" in kw:
                s.tick(kw["P"])
            s.upsert([5], _junk(am, 1))  # (staged: a refused restore drains nothing)
            s.post_result([3], [2])
            pair.append(s)
        t, c = pair
        try:
            with pytest.raises(am.AmError) as e:
                t.restore(b)
            assert e.value.code == code, (what, e.value.code)
            for s in pair:
                probe.append((s.tick(T + 60, mode=CATCH), s.read_range(0, 8)))
            ((ti, ta, ts), tc), ((ci, ca, cs), cc) = probe
            assert ti.tolist() == ci.tolist() and ta.tolist() == ca.tolist() and ts == cs, what
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(tc[name], cc[name], err_msg=f"{what}: {name}")
        finally:
            t.close()
            c.close()
    # AM_E_NOSPACE: the size the call needs, then a blob no longer than it
    s = am.Sweep(capacity=n)
    try:
        s.upsert(np.arange(n), recs)
        need = ctypes.c_uint64(0)
        buf = np.zeros(10, np.uint8)
        assert s._lib.am_sweep_checkpoint(s._h, 0, n, buf.ctypes.data, 10, ctypes.byref(need)) == am.AM_E_NOSPACE
        b = s.checkpoint(0, n)
        # (the size it needs has room for the names of every zone registered in the process)
        assert fmt.sections(n, am.CKPT_TIMEOUTS)[1] + 8 * len(ZONE_NAMES) <= need.value and len(b) <= need.value
        assert fmt.read(b)["checksum_ok"]
        assert am.checkpoint_info(b)["prev_tick"] is None and am.checkpoint_info(b)["switches"] == am.CKPT_TIMEOUTS
        with pytest.raises(am.AmError) as e:
            am.checkpoint_info(b[:100])
        assert e.value.code == am.AM_E_INVAL
    finally:
        s.close()


CHILD_FULL = r"""
import ctypes as C, importlib, os, sys
sys.path.insert(0, {root!r})
am = importlib.import_module("active-monitor_b200")
blob = open({path!r}, "rb").read()
info = am.checkpoint_info(blob)
names = set({names!r})
zones = sorted(os.path.relpath(os.path.join(d, f), "/usr/share/zoneinfo") for d, _, fs in os.walk("/usr/share/zoneinfo")
               for f in fs)
rc = am.AM_OK
for z in zones:
    if z in names or "/" not in z or z.startswith(("posix/", "right/")):
        continue
    i = C.c_int32()
    rc = am.load().am_tz_lookup(z.encode(), len(z), C.byref(i))
    if rc == am.AM_E_UNSUPPORTED:
        break
assert rc == am.AM_E_UNSUPPORTED, "the registry did not fill"
s = am.Sweep(capacity=info["n"])
s.set_hold_in_flight(True)
try:
    s.restore(blob)
    print("restored")
except am.AmError as e:
    assert e.code == am.AM_E_UNSUPPORTED, e.code
    assert (s.read_range(0, info["n"])["flags"] == am.F_TOMBSTONE).all()
    print("ok unsupported")
"""


def test_refusal_256th_zone(am, zmap):
    """a blob whose zones do not fit a full registry (in a child process: the registry is process-wide)"""
    if not os.path.isdir("/usr/share/zoneinfo"):
        pytest.skip("no zoneinfo directory")
    rng = np.random.default_rng(8)
    n = 200
    s = am.Sweep(capacity=n)
    s.set_hold_in_flight(True)
    try:
        s.upsert(np.arange(n), _records(am, zmap, rng, n, T_PARIS, False))
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "blob")
            with open(path, "wb") as f:
                f.write(s.checkpoint(0, n))
            assert fmt.read(open(path, "rb").read())["n_zones"] > 0
            code = CHILD_FULL.format(root=ROOT, path=path, names=list(fmt.read(open(path, "rb").read())["zones"].values()))
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0 and "ok unsupported" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    finally:
        s.close()


def test_full_size(am):
    """10 M config-5 records with both holds and a tenth with workflow timeouts: simulate, checkpoint, restore, go on;
    bit-exact against the uninterrupted handle"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import run_sim
    n, S = 10_000_000, 1800
    cols, sl, recs = run_sim.population(am, n, 3)
    handles = []
    for _ in range(2):
        s = am.Sweep(capacity=n)
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        s.set_hold_remedy(True)
        s.upsert(sl, recs)
        handles.append(s)
    a, b = handles
    try:
        T0 = run_sim.amgen.T0_DAY_START
        ra, sa = a.simulate(T0, 2 * S, BLOCKED, 3, run_sim.PARAMS)
        rb, sb = b.simulate(T0, S, BLOCKED, 3, run_sim.PARAMS)
        blob = b.checkpoint(0, n)
        b.close()
        b = _fresh(am, n, 0, am.checkpoint_info(blob))
        handles[1] = b
        b.restore(blob)
        del blob
        rc, sc = b.simulate(T0 + S, S, BLOCKED, 3, run_sim.PARAMS)
        np.testing.assert_array_equal(np.concatenate([rb, rc]), ra)
        np.testing.assert_array_equal(np.concatenate([sb, sc]), sa)
        assert sa["n_in_flight"].max() > 0 and sa["n_timed_out"].sum() > 0
        ga, gb = a.read_range(0, n), b.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(gb[name], ga[name], err_msg=name)
        np.testing.assert_array_equal(b.in_flight(0, n), a.in_flight(0, n))
        np.testing.assert_array_equal(b.remedy_in_flight(0, n), a.remedy_in_flight(0, n))
        for T in range(T0 + 2 * S, T0 + 2 * S + 3):
            ia, aa, sta = a.tick(T)
            ib, ab, stb = b.tick(T)
            assert sta == stb and np.array_equal(ia, ib) and np.array_equal(aa, ab)
    finally:
        for s in handles:
            s.close()
