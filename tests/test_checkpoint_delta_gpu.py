"""Delta checkpoints: am_sweep_checkpoint_chain / _delta, am_checkpoint_delta_info and am_sweep_restore_delta.  A walk
of random calls and ticks on a source handle takes a chain's root and deltas every few steps; a standby restores the
root and applies each delta.  After every link the delta's slots equal the numpy diff of two full blobs of the source
(the previous link's and one taken right after the delta), the numpy reader (tests/checkpoint_delta_format.py) applied
to the previous full arrays gives the new full blob's, and a full checkpoint of the standby is byte for byte the
source's.  With the handle model (tests/handle_model.py) the walk then goes on with the standby against the unchanged
model.  Also: a range over several 8192-slot groups that ends inside one, a delta with no changed slot,
AM_E_NOSPACE, switches toggled between links, a chain over a sub-range at a base past 2^32, two shards' chains applied
to one standby in both orders, a zone registered after the root, every refusal, the launch counts, and 10 M records
(GPU only)."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest

import checkpoint_delta_format as dfmt
from adversarial import ZONE_NAMES, ZoneMap
from handle_pair import Pair, emulated
from test_checkpoint_gpu import SWITCHES, T_PARIS, _fresh, _junk, _records

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CATCH, BLOCKED = 0x8, 0x4
WALKS = dict(SWITCHES, hold_budget=dict(hold=True))  # (+ a finite submit budget: the waiting-second section)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _standby(am, root, capacity, shard_base, budget=None):
    s = _fresh(am, capacity, shard_base, am.checkpoint_info(root))
    if budget is not None:
        s.set_submit_budget(budget)
    s.restore(root)
    return s


def _check_link(am, src, sb, prev_full, delta, n_changed, first, n, sb_first=None):
    """the delta against the numpy diff of the previous link's full blob and the source's state now; the reader's
    apply against the new full blob; the standby's full checkpoint against the source's.  Returns the new full blob."""
    full = src.checkpoint(first, n)
    a, b = dfmt.read_full(prev_full), dfmt.read_full(full)
    d = dfmt.read(delta)
    assert d["checksum_ok"] and b["checksum_ok"]
    assert d["n_changed"] == n_changed == len(d["offsets"])
    np.testing.assert_array_equal(d["offsets"], dfmt.diff(a, b))
    got = dfmt.apply(a, d)
    for name, *_ in dfmt.sections(0, b["switches"])[0]:
        np.testing.assert_array_equal(got[name], b[name], err_msg=name)
    for k in ("swept_end", "prev_tick", "seed", "zones", "first_global", "n", "switches"):
        assert got[k] == b[k], k
    info = am.checkpoint_delta_info(delta)
    assert info["n_changed"] == n_changed and info["bytes"] == len(delta) and info["checksum"] == d["checksum"]
    sb.restore_delta(delta)
    assert sb.checkpoint(first if sb_first is None else sb_first, n) == full
    return full


def _random_call(am, zmap, src, p, rng, T, timeouts, n):
    c = rng.integers(0, 6)
    tgt = p or src
    hwm = p.m.hwm if p else src.size
    if c == 0:
        sl = rng.choice(n, rng.integers(1, 40), replace=True)
        tgt.upsert(sl, _records(am, zmap, rng, len(sl), T, timeouts))
    elif c == 1:
        tgt.remove(rng.choice(n, rng.integers(1, 10), replace=False))
    elif c in (2, 3) and hwm:
        sl = rng.choice(hwm, rng.integers(1, 80), replace=True)
        ph, rp = rng.integers(0, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8)
        if p:
            p.post(sl, ph, rp)
        else:
            src.post_result(sl, ph, rp)


def _tick(src, p, T, mode):
    return p.tick(T, mode=mode) if p else src.tick(T, mode=mode)


@pytest.mark.parametrize("timeouts", [False, True], ids=["no_timeouts", "timeouts"])
@pytest.mark.parametrize("switches", list(WALKS))
def test_walk(am, zmap, switches, timeouts):
    rng = np.random.default_rng(zlib.crc32(f"delta {switches} {timeouts}".encode()))
    n = 700
    T = T_PARIS
    budget = 5 if switches == "hold_budget" else None
    p = None if budget else Pair(am, zmap, n, seed=7, every_slot=False, **WALKS[switches])
    src = p.s if p else am.Sweep(capacity=n)
    sb = None
    try:
        if budget:
            src.set_hold_in_flight(True)
            src.set_seed(7)
            src.set_submit_budget(budget)
        recs = _records(am, zmap, rng, n - 37, T, timeouts)
        (p or src).upsert(np.arange(n - 37), recs)
        _tick(src, p, T, 0)
        root = src.checkpoint_chain(0, n)
        assert root == src.checkpoint(0, n)
        sb = _standby(am, root, n, 0, budget)
        prev, links, nonzero = root, 0, 0
        next_link = 1
        for step in range(30):
            for _ in range(rng.integers(0, 3)):
                _random_call(am, zmap, src, p, rng, T, timeouts, n)
            T += int(rng.choice([1, 1, 2, 7, 30, 60]))
            _tick(src, p, T, CATCH if rng.random() < 0.3 else 0)
            if step + 1 == next_link:
                if rng.random() < 0.4:  # (staged before the delta: it drains them)
                    _random_call(am, zmap, src, p, rng, T, timeouts, n)
                    _random_call(am, zmap, src, p, rng, T, timeouts, n)
                delta, k = src.checkpoint_delta()
                prev = _check_link(am, src, sb, prev, delta, k, 0, n)
                links += 1
                nonzero += k > 0
                next_link += int(rng.integers(1, 6))
        delta, k = src.checkpoint_delta()  # (the last link: the standby catches up with the source)
        _check_link(am, src, sb, prev, delta, k, 0, n)
        assert links >= 6 and nonzero >= 4
        # fail over: the standby goes on in the source's place
        if p:
            p.s.close()
            p.s = sb
            sb = None
            for k in range(1, 6):
                _random_call(am, zmap, None, p, rng, T, timeouts, n)
                p.tick(T + k, mode=CATCH if k == 1 else 0)
        else:
            for k in range(1, 6):
                want, got = src.tick(T + 60 * k, mode=CATCH), sb.tick(T + 60 * k, mode=CATCH)
                assert want[0].tolist() == got[0].tolist() and want[1].tolist() == got[1].tolist() and want[2] == got[2]
            assert sb.checkpoint(0, n) == src.checkpoint(0, n)
    finally:
        (p or src).close()
        if sb:
            sb.close()


def test_multi_group_range(am, zmap):
    """a chain whose range starts off a word edge, spans several 8192-slot groups and ends inside a group (the diff's
    per-group counts, the cross-group scan and compaction, the pack at ranks past a group), through small deltas and
    one in which every swept slot changed"""
    rng = np.random.default_rng(11)
    n, T = 3 * 8192 + 1234, T_PARIS
    first, m = 37, 3 * 8192 + 1234 - 74
    s = _hold_handle(am, zmap, rng, n - 500, T, capacity=n)  # (the last 500 slots never swept)
    root = s.checkpoint_chain(first, m)
    sb = _standby(am, root, n, 0)
    try:
        prev, sizes = root, []
        for k in range(6):
            if k == 3:  # every swept slot upserted again
                s.upsert(np.arange(n - 500), _records(am, zmap, rng, n - 500, T, True))
            else:
                s.post_result(rng.choice(n - 500, 300), rng.integers(0, 3, 300).astype(np.uint8))
                s.upsert(rng.choice(n, 25), _records(am, zmap, rng, 25, T, True))
            T += int(rng.choice([1, 7, 60]))
            s.tick(T)
            delta, c = s.checkpoint_delta()
            prev = _check_link(am, s, sb, prev, delta, c, first, m)
            sizes.append(c)
            offs = dfmt.read(delta)["offsets"]
            assert len(np.unique(offs // 8192)) >= 3, (k, c)  # (changed slots in several groups)
        assert max(sizes) > 2 * 8192 and min(sizes) > 0, sizes
    finally:
        s.close()
        sb.close()


def test_full_size(am):
    """10 M config-5 records with both holds and a tenth with workflow timeouts: a simulated half hour, a chain's root,
    then deltas after simulated periods of 1, 10 and 60 s applied to a standby.  Each delta's slots are the numpy diff
    of the source's full blobs; the standby's full checkpoint is the source's, and it then ticks bit-exact against it."""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import run_sim
    n, S = 10_000_000, 1800
    cols, sl, recs = run_sim.population(am, n, 3)
    src = am.Sweep(capacity=n)
    sb = None
    try:
        src.load_range(0, cols)
        src.set_hold_in_flight(True)
        src.set_hold_remedy(True)
        src.upsert(sl, recs)
        T = run_sim.amgen.T0_DAY_START
        rows, sims = src.simulate(T, S, BLOCKED, 3, run_sim.PARAMS)
        assert sims["n_in_flight"].max() > 0 and sims["n_timed_out"].sum() > 0
        T += S
        root = src.checkpoint_chain(0, n)
        info = am.checkpoint_info(root)
        assert info["switches"] == am.CKPT_HOLD | am.CKPT_REMEDY | am.CKPT_TIMEOUTS
        sb = _fresh(am, n, 0, info)
        sb.restore(root)
        prev = dfmt.read_full(root)
        del root
        for period in (1, 10, 60):
            src.simulate(T, period, BLOCKED, 3, run_sim.PARAMS)
            T += period
            delta, k = src.checkpoint_delta()
            full = src.checkpoint(0, n)
            cur = dfmt.read_full(full)
            want = dfmt.diff(prev, cur)
            d = dfmt.read(delta)
            assert d["checksum_ok"] and k == d["n_changed"] == len(want) > 0, (period, k, len(want))
            np.testing.assert_array_equal(d["offsets"], want, err_msg=f"period {period}")
            sb.restore_delta(delta)
            prev = cur
            del delta, d
        assert sb.checkpoint(0, n) == full
        del full, prev, cur
        for t in range(T, T + 3):
            ia, aa, sta = src.tick(t)
            ib, ab, stb = sb.tick(t)
            assert sta == stb and np.array_equal(ia, ib) and np.array_equal(aa, ab), t
    finally:
        src.close()
        if sb:
            sb.close()


def _hold_handle(am, zmap, rng, n, T, shard_base=0, capacity=None, timeouts=True):
    s = am.Sweep(capacity=capacity or n, shard_base=shard_base)
    s.set_hold_in_flight(True)
    s.upsert(np.arange(n), _records(am, zmap, rng, n, T, timeouts))
    s.tick(T)
    return s


def test_zero_change_delta(am, zmap):
    """a chain over slots nothing writes: a tick moves only P and the seed, and the delta carries no slot"""
    rng = np.random.default_rng(1)
    n, T = 400, T_PARIS
    s = _hold_handle(am, zmap, rng, n - 100, T, capacity=n)
    root = s.checkpoint_chain(n - 100, 100)
    sb = _standby(am, root, n, 0)
    try:
        s.set_seed(99)
        s.tick(T + 5)
        delta, k = s.checkpoint_delta()
        info = am.checkpoint_delta_info(delta)
        assert k == 0 and info["n_changed"] == 0 and info["prev_tick"] == T + 5 and info["parent_prev_tick"] == T
        assert info["seq"] == 1 and info["seed"] == 99
        _check_link(am, s, sb, root, delta, k, n - 100, 100)
        assert am.checkpoint_info(sb.checkpoint(n - 100, 100))["prev_tick"] == T + 5
        delta2, k2 = s.checkpoint_delta()  # (nothing at all since the last link)
        assert k2 == 0 and am.checkpoint_delta_info(delta2)["seq"] == 2
        sb.restore_delta(delta2)
    finally:
        s.close()
        sb.close()


def test_nospace_commits_nothing(am, zmap):
    rng = np.random.default_rng(2)
    n, T = 500, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    root = s.checkpoint_chain(0, n)
    sb = _standby(am, root, n, 0)
    try:
        s.post_result(np.arange(0, n, 3), np.full(len(range(0, n, 3)), 2, np.uint8))
        s.tick(T + 1)
        need, changed = ctypes.c_uint64(0), ctypes.c_uint64(0)
        buf = np.zeros(16, np.uint8)
        rc = s._lib.am_sweep_checkpoint_delta(s._h, buf.ctypes.data, 16, ctypes.byref(need), ctypes.byref(changed))
        assert rc == am.AM_E_NOSPACE and need.value > 16
        with pytest.raises(am.AmError) as e:
            s.checkpoint_delta(cap=need.value - 8)
        assert e.value.code == am.AM_E_NOSPACE
        s.upsert([1], _records(am, zmap, rng, 1, T, True))
        delta, k = s.checkpoint_delta()
        assert am.checkpoint_delta_info(delta)["seq"] == 1
        _check_link(am, s, sb, root, delta, k, 0, n)  # (the slots of the refused calls, and the upsert since)
        assert k > n // 3
    finally:
        s.close()
        sb.close()


def test_switches_toggled_between_links(am, zmap):
    rng = np.random.default_rng(3)
    n, T = 300, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T, timeouts=False)
    try:
        root = s.checkpoint_chain(0, n)
        s.set_track_changes(True)
        with pytest.raises(am.AmError) as e:
            s.checkpoint_delta()
        assert e.value.code == am.AM_E_INVAL
        root = s.checkpoint_chain(0, n)  # a new chain works
        sb = _standby(am, root, n, 0)
        s.tick(T + 3)
        delta, k = s.checkpoint_delta()
        _check_link(am, s, sb, root, delta, k, 0, n)
        # the timeout state appears through an upsert: the switches differ from the root's
        recs = _records(am, zmap, rng, 1, T, False)
        recs["wf_timeout"] = 30
        s.upsert([4], recs)
        with pytest.raises(am.AmError) as e:
            s.checkpoint_delta()
        assert e.value.code == am.AM_E_INVAL
        root = s.checkpoint_chain(0, n)
        assert am.checkpoint_info(root)["switches"] & am.CKPT_TIMEOUTS
        sb.close()
        sb = _standby(am, root, n, 0)
        s.tick(T + 4)
        delta, k = s.checkpoint_delta()
        _check_link(am, s, sb, root, delta, k, 0, n)
        sb.close()
    finally:
        s.close()
    with pytest.raises(am.AmError) as e:  # (no chain at all)
        t = am.Sweep(capacity=8)
        try:
            t.checkpoint_delta()
        finally:
            t.close()
    assert e.value.code == am.AM_E_INVAL


def test_sub_range_past_2_32(am, zmap):
    """a chain over a sub-range of a shard whose base is past 2^32, applied to a standby with another base and a
    larger capacity"""
    rng = np.random.default_rng(4)
    n, T = 900, T_PARIS
    base = (1 << 32) + 1000
    s = _hold_handle(am, zmap, rng, n, T, shard_base=base)
    a, m = 211, 433
    root = s.checkpoint_chain(a, m)
    assert am.checkpoint_info(root)["first_global"] == base + a
    sb = _standby(am, root, 2000, base - 500)
    try:
        prev = root
        for k in range(4):
            s.post_result(rng.choice(n, 60), rng.integers(0, 3, 60).astype(np.uint8))
            s.tick(T + 1 + k)
            delta, c = s.checkpoint_delta()
            info = am.checkpoint_delta_info(delta)
            assert info["first_global"] == base + a and info["n"] == m
            prev = _check_link(am, s, sb, prev, delta, c, a, m, sb_first=a + 500)
            assert c > 0  # (the standby's local slots are shifted by 500)
    finally:
        s.close()
        sb.close()


def test_two_shards_one_standby(am, zmap):
    """two source shards' chains, their deltas taken at the same ticks, applied to one standby in both orders"""
    rng = np.random.default_rng(5)
    n, T = 400, T_PARIS
    srcs = [_hold_handle(am, zmap, rng, n, T, shard_base=b) for b in (0, n)]
    try:
        roots = [s.checkpoint_chain(0, n) for s in srcs]
        for order in ((0, 1), (1, 0)):
            sb = am.Sweep(capacity=2 * n)
            sb.set_hold_in_flight(True)
            for r in roots:
                sb.restore(r)
            for s in srcs:  # (both sources tick at the same second)
                s.post_result(rng.choice(n, 40), rng.integers(0, 3, 40).astype(np.uint8))
                s.tick(T + 10 * (order[0] + 1))
            deltas = [s.checkpoint_delta()[0] for s in srcs]
            for k in order:
                sb.restore_delta(deltas[k])
            for k, s in enumerate(srcs):
                full, mine = s.checkpoint(0, n), sb.checkpoint(k * n, n)
                want, got = dfmt.read_full(full), dfmt.read_full(mine)
                for name, *_ in dfmt.sections(0, want["switches"])[0]:
                    np.testing.assert_array_equal(got[name], want[name], err_msg=f"{order} {k} {name}")
                for f in ("prev_tick", "seed", "swept_end", "first_global"):  # (P: the parent's for one, its own for the other)
                    assert got[f] == want[f], (order, k, f)
                assert mine == full, (order, k)
            roots = [s.checkpoint_chain(0, n) for s in srcs]  # (the next order starts from fresh roots)
            sb.close()
    finally:
        for s in srcs:
            s.close()


CHILD = """
import json, sys
sys.path.insert(0, {root!r})
sys.path.insert(0, {root!r} + "/tests")
import importlib
am = importlib.import_module("active-monitor_b200")
ids = {{z: am.tz_lookup(z) for z in {names!r}}}
root, delta = open({path!r} + ".root", "rb").read(), open({path!r} + ".delta", "rb").read()
info = am.checkpoint_info(root)
s = am.Sweep(capacity=info["n"])
s.set_hold_in_flight(True)
s.restore(root)
s.restore_delta(delta)
out = {{"ids": ids, "ticks": []}}
for T in {ticks!r}:
    i, a, st = s.tick(T, mode=8)
    out["ticks"].append([i.tolist(), a.tolist(), st])
print(json.dumps(out))
"""


def test_zone_registered_after_the_root(am, zmap):
    """a delta whose records use a zone the root's do not, applied in a process that registered the zones in another
    order, ticks as the source"""
    rng = np.random.default_rng(9)
    n = 300
    T = 1792890000 - 181
    s = am.Sweep(capacity=n)
    s.set_hold_in_flight(True)
    try:
        recs = _records(am, zmap, rng, n, T, True)
        flags = recs["flags"]
        bound = (flags & np.uint32(7)) == am.KIND_CRON_SPEC
        zones_used = set((flags[bound] >> np.uint32(24)).tolist()) - {0}
        spare = [z for z in ZONE_NAMES if zmap.ids[z] not in zones_used]
        assert bound.any() and spare
        late = spare[0]
        recs["flags"] = np.where(bound & ((flags >> np.uint32(24)) == np.uint32(zmap.ids[late])), flags & np.uint32(0xFFFFFF), flags)
        s.upsert(np.arange(n), recs)
        s.tick(T)
        root = s.checkpoint_chain(0, n)
        assert late not in dfmt.read_full(root)["zones"].values()
        k = int(np.flatnonzero(bound)[0])
        one = recs[k:k + 1].copy()
        one["flags"] = (one["flags"] & np.uint32(0xFFFFFF)) | np.uint32(zmap.ids[late] << 24)
        s.upsert([k], one)
        delta, c = s.checkpoint_delta()
        assert c >= 1 and late in dfmt.read(delta)["zones"].values()
        ticks = [T + 60 * j + 1 for j in range(1, 7)]
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "blob")
            open(path + ".root", "wb").write(root)
            open(path + ".delta", "wb").write(delta)
            code = CHILD.format(root=ROOT, names=list(reversed(ZONE_NAMES)), path=path, ticks=ticks)
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        child = json.loads(r.stdout.strip().splitlines()[-1])
        assert any(child["ids"][z] != zmap.ids[z] for z in child["ids"])
        for T, (ci, ca, cs) in zip(ticks, child["ticks"]):
            i, a, st = s.tick(T, mode=CATCH)
            assert ci == i.tolist() and ca == a.tolist() and cs == st, T
    finally:
        s.close()


def _flip(blob, at):
    b = bytearray(blob)
    b[at] ^= 1
    return bytes(b)


def test_refusals_change_nothing(am, zmap):
    """every refused delta leaves the standby as it was: a full checkpoint before and after is the same"""
    rng = np.random.default_rng(6)
    n, T = 300, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    other = _hold_handle(am, zmap, np.random.default_rng(7), n, T)
    try:
        root = s.checkpoint_chain(0, n)
        other.checkpoint_chain(0, n)
        s.post_result(rng.choice(n, 50), np.full(50, 2, np.uint8))
        s.tick(T + 1)
        d1, k1 = s.checkpoint_delta()
        s.post_result(rng.choice(n, 50), np.full(50, 1, np.uint8))
        s.tick(T + 2)
        d2, k2 = s.checkpoint_delta()
        other.tick(T + 1)
        foreign, _ = other.checkpoint_delta()
        assert k1 > 0 and k2 > 0
        r1 = dfmt.read(d1)
        m = r1["n_changed"]
        secs, end = dfmt.sections(m, r1["switches"], dfmt.start_of(m))
        bad_off = bytearray(d1)
        bad_off[dfmt.HEADER:dfmt.HEADER + 4] = (n + 5).to_bytes(4, "little")
        cases = [("skipped link", d2, {}), ("foreign chain", foreign, {}), ("truncated", d1[:-8], {}),
                 ("no root", d1, dict(no_root=True)), ("ticked", d1, dict(tick=True)),
                 ("outside the shard", d1, dict(capacity=n - 1)),
                 ("offset section", _flip(d1, dfmt.HEADER + 1), {}),
                 ("offset past n, resealed", _reseal(bytes(bad_off)), {})]
        cases += [(f"section {name}", _flip(d1, off), {}) for name, dt, off, nbytes in secs if nbytes]
        for what, b, kw in cases:
            sb = am.Sweep(capacity=kw.get("capacity", n))
            sb.set_hold_in_flight(True)
            try:
                if not kw.get("no_root") and "capacity" not in kw:
                    sb.restore(root)
                if kw.get("tick"):
                    sb.tick(T + 1)
                before = sb.checkpoint(0, sb.capacity)
                with pytest.raises(am.AmError) as e:
                    sb.restore_delta(b)
                want = am.AM_E_RANGE if "capacity" in kw else am.AM_E_INVAL
                assert e.value.code == want, (what, e.value.code)
                assert sb.checkpoint(0, sb.capacity) == before, what
            finally:
                sb.close()
        # a link applied twice
        sb = _standby(am, root, n, 0)
        try:
            sb.restore_delta(d1)
            before = sb.checkpoint(0, n)
            with pytest.raises(am.AmError) as e:
                sb.restore_delta(d1)
            assert e.value.code == am.AM_E_INVAL and sb.checkpoint(0, n) == before
            sb.restore_delta(d2)
            assert sb.checkpoint(0, n) == s.checkpoint(0, n)
        finally:
            sb.close()
        # a delta is not a full blob, and a full blob is not a delta
        for fn in (lambda: am.checkpoint_info(d1), lambda: am.checkpoint_delta_info(root)):
            with pytest.raises(am.AmError) as e:
                fn()
            assert e.value.code == am.AM_E_INVAL
        sb = am.Sweep(capacity=n)
        sb.set_hold_in_flight(True)
        try:
            with pytest.raises(am.AmError) as e:
                sb.restore(d1)
            assert e.value.code == am.AM_E_INVAL
        finally:
            sb.close()
    finally:
        s.close()
        other.close()


def _reseal(delta):
    """a copy of a delta with its checksum recomputed from the documented rule (for edits made on purpose)"""
    b = bytearray(delta)
    b[dfmt.fmt.CHECKSUM_AT:dfmt.fmt.CHECKSUM_AT + 8] = _sum_of(delta).to_bytes(8, "little")
    assert dfmt.read(bytes(b))["checksum_ok"]
    return bytes(b)


def _sum_of(delta):
    raw = np.frombuffer(delta, dtype=np.uint8)
    hd = raw[:dfmt.HEADER].view(dfmt.HEADER_FIELDS)[0]
    m = int(hd["n_changed"])
    offs = raw[dfmt.HEADER:dfmt.HEADER + 4 * m].view("<u4")
    s = dfmt.fmt._sum(dfmt.fmt.mix((np.uint64(dfmt.HEADER) + np.arange(m, dtype=np.uint64) * np.uint64(4)) *
                                   np.uint64(8), offs.astype(np.uint64)))
    secs, end = dfmt.sections(m, int(hd["switches"]), dfmt.start_of(m))
    s += dfmt._elements(raw, secs, m)[1]
    s += dfmt._header_and_zones(raw, end, hd, int(hd["n_zones"]))[2]
    return s % (1 << 64)


def test_launch_counts(am, zmap):
    rng = np.random.default_rng(8)
    n, T = 300, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    try:
        root = s.checkpoint_chain(0, n)
        sb = _standby(am, root, n, 0)
        c0 = s.launch_count
        d0, k0 = s.checkpoint_delta(cap=1 << 20)  # nothing staged, nothing changed: diff, scan, compaction, pack
        assert k0 == 0 and s.launch_count - c0 == 4
        s.tick(T + 1)
        c0 = s.launch_count
        d1, k1 = s.checkpoint_delta(cap=1 << 20)  # ... and the commit
        assert k1 > 0 and s.launch_count - c0 == 5
        b0 = sb.launch_count
        sb.restore_delta(d0)
        assert sb.launch_count == b0
        sb.restore_delta(d1)  # offsets and sections verified, scatter, plane rebuild
        assert sb.launch_count - b0 == 4
        sb.close()
    finally:
        s.close()
    quiet = am.Sweep(capacity=n)  # a handle that never starts a chain launches nothing for one
    try:
        quiet.upsert(np.arange(10), _junk(am, 10))
        quiet.tick(T)
        c0 = quiet.launch_count
        quiet.checkpoint(0, n)
        assert quiet.launch_count - c0 == 1
    finally:
        quiet.close()
