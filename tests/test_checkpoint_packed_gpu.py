"""Packed checkpoints: am_sweep_set_checkpoint_packing, and format version 2 through am_sweep_checkpoint, _chain,
_delta, both restores and both info calls.  The numpy decoder of tests/checkpoint_packed_format.py turns every packed
blob into version-1 bytes: a packed full blob is byte for byte the raw one taken at the same point, and a packed delta
reads as a delta whose slots are the numpy diff of the source's full blobs.  Walks of random calls and ticks under
every switch combination (tests/handle_pair.py) take chains whose roots and links are packed or raw at random; a
standby follows them, its full checkpoints (raw and packed) equal the source's, and after a failover it goes on
against the model.  Also: columns built so that each mode wins, 64-bit extremes, ranges that start inside a word or
hold one slot, a base past 2^32, the size bound, every refusal of a malformed packed blob (nothing changed, nothing
drained), the launch counts, and 10 M records (GPU only)."""
import ctypes
import zlib

import numpy as np
import pytest

import checkpoint_packed_format as pf
from adversarial import ZoneMap
from handle_pair import Pair, emulated
from test_checkpoint_delta_gpu import WALKS, _check_link, _flip, _hold_handle, _random_call, _standby, _tick
from test_checkpoint_gpu import T_PARIS, _fresh, _junk, _records

pytestmark = pytest.mark.gpu

BLOCKED = 0x4


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _full(h, first, n, packed):
    """a full checkpoint of h in one encoding; the packing setting as it was before"""
    was = getattr(h, "_packing", False)
    h.set_checkpoint_packing(packed)
    try:
        return h.checkpoint(first, n)
    finally:
        h.set_checkpoint_packing(was)


def _both(am, h, first, n):
    """the raw and the packed full checkpoint of h at one point: the packed one decodes to the raw one, within the
    bound, and reports version 2 and its own length"""
    raw, packed = _full(h, first, n, False), _full(h, first, n, True)
    assert pf.decode(packed) == raw
    assert len(packed) <= pf.bound(len(raw), packed)
    info, rinfo = am.checkpoint_info(packed), am.checkpoint_info(raw)
    assert info["version"] == 2 and rinfo["version"] == 1 and info["bytes"] == len(packed)
    assert {k: v for k, v in info.items() if k not in ("version", "bytes")} == \
        {k: v for k, v in rinfo.items() if k not in ("version", "bytes")}
    return raw, packed


def _check_packed_link(am, src, sb, prev_full, delta, k, first, n):
    """_check_link on the version-1 bytes the delta decodes to, with the packed delta applied to the standby; both
    encodings of the standby's full checkpoint against the source's"""
    packed = am.checkpoint_delta_info(delta)["version"] == 2
    v1 = pf.decode(delta) if packed else delta
    if packed:
        info, rinfo = am.checkpoint_delta_info(delta), am.checkpoint_delta_info(v1)
        assert info["bytes"] == len(delta) and len(delta) <= pf.bound(len(v1), delta)
        assert {k: v for k, v in info.items() if k not in ("version", "bytes")} == \
            {k: v for k, v in rinfo.items() if k not in ("version", "bytes")}

    class Raw:  # raw full checkpoints of a handle, and the standby applies the blob as the source wrote it
        def __init__(self, h):
            self.h = h

        def restore_delta(self, _):
            self.h.restore_delta(delta)

        def checkpoint(self, a, b):
            return _full(self.h, a, b, False)
    full = _check_link(am, Raw(src), Raw(sb), prev_full, v1, k, first, n)
    assert _full(sb, first, n, True) == _full(src, first, n, True)  # (determinism: the same state, the same bytes)
    return full


@pytest.mark.parametrize("timeouts", [False, True], ids=["no_timeouts", "timeouts"])
@pytest.mark.parametrize("switches", list(WALKS))
def test_walk(am, zmap, switches, timeouts):
    rng = np.random.default_rng(zlib.crc32(f"packed {switches} {timeouts}".encode()))
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
        (p or src).upsert(np.arange(n - 37), _records(am, zmap, rng, n - 37, T, timeouts))
        _tick(src, p, T, 0)
        raw, packed = _both(am, src, 0, n)
        root_packed = bool(rng.integers(0, 2))
        src.set_checkpoint_packing(root_packed)
        root = src.checkpoint_chain(0, n)
        assert root == (packed if root_packed else raw)
        sb = _standby(am, root, n, 0, budget)
        assert sb.checkpoint(0, n) == raw
        prev, kinds = raw, set()
        next_link = 1
        for step in range(24):
            for _ in range(rng.integers(0, 3)):
                _random_call(am, zmap, src, p, rng, T, timeouts, n)
            T += int(rng.choice([1, 1, 2, 7, 30, 60]))
            _tick(src, p, T, 0x8 if rng.random() < 0.3 else 0)
            if step + 1 == next_link:
                link_packed = bool(rng.integers(0, 2)) if step > 2 else step % 2 == 0
                src.set_checkpoint_packing(link_packed)
                delta, k = src.checkpoint_delta()
                prev = _check_packed_link(am, src, sb, prev, delta, k, 0, n)
                kinds.add((root_packed, link_packed))
                next_link += int(rng.integers(1, 4))
        assert {r for r, _ in kinds} == {root_packed} and len(kinds) == 2, kinds  # (both kinds of link)
        # restore equivalence: a fresh handle restored from the packed blob checkpoints as the source does
        raw, packed = _both(am, src, 0, n)
        t = _fresh(am, n, 0, am.checkpoint_info(packed))
        if budget:
            t.set_submit_budget(budget)
        t.restore(packed)
        assert t.checkpoint(0, n) == raw and _full(t, 0, n, True) == packed
        sb.close()
        sb = t
        # fail over: the handle restored from the packed blob goes on in the source's place
        if p:
            p.s.close()
            p.s = sb
            sb = None
            for k in range(1, 6):
                _random_call(am, zmap, None, p, rng, T, timeouts, n)
                p.tick(T + k, mode=0x8 if k == 1 else 0)
        else:
            for k in range(1, 6):
                want, got = src.tick(T + 60 * k, mode=0x8), sb.tick(T + 60 * k, mode=0x8)
                assert want[0].tolist() == got[0].tolist() and want[1].tolist() == got[1].tolist() and want[2] == got[2]
            assert sb.checkpoint(0, n) == _full(src, 0, n, False)
    finally:
        (p or src).close()
        if sb:
            sb.close()


def test_mixed_chains(am, zmap):
    """one source, three chains over the same range: packed root and links, raw root with packed links, packed root
    with raw links; each standby's full checkpoint equals the source's in both encodings"""
    rng = np.random.default_rng(21)
    n, T = 2500, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    try:
        for root_packed, links_packed in ((True, True), (False, True), (True, False)):
            s.set_checkpoint_packing(root_packed)
            root = s.checkpoint_chain(0, n)
            assert am.checkpoint_info(root)["version"] == (2 if root_packed else 1)
            sb = _standby(am, root, n, 0)
            try:
                prev = _full(s, 0, n, False)
                for k in range(4):
                    s.post_result(rng.choice(n, 200), rng.integers(0, 3, 200).astype(np.uint8))
                    s.upsert(rng.choice(n, 20), _records(am, zmap, rng, 20, T, True))
                    T += int(rng.choice([1, 7, 60]))
                    s.tick(T)
                    s.set_checkpoint_packing(links_packed)
                    delta, c = s.checkpoint_delta()
                    assert am.checkpoint_delta_info(delta)["version"] == (2 if links_packed else 1)
                    prev = _check_packed_link(am, s, sb, prev, delta, c, 0, n)
                assert sb.checkpoint(0, n) == _full(s, 0, n, False)
            finally:
                sb.close()
    finally:
        s.close()


def _adversarial_cols(am, rng, n):
    """columns whose blocks each favour one mode, with 64-bit extremes next to real values"""
    rc, r = am.classify(repeat_after_sec=60, finished_at=0)
    assert rc == 0
    cols = am.records_to_columns(np.repeat(r, n))
    u64 = lambda a: np.asarray(a, np.uint64)
    cols["minute"] = u64(rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + u64(rng.integers(0, 2, n)))  # RAW, width 64
    cols["hour"] = u64(np.full(n, 0xFFFFFF))  # CONST
    cols["dom"] = u64((1 << 40) + rng.integers(0, 1 << 12, n))  # FOR
    dow = np.zeros(n, np.uint64)  # SPARSE: mostly 0
    hit = rng.random(n) < 0.02
    dow[hit] = u64((1 << 50) + rng.integers(0, 1 << 20, hit.sum()))
    cols["dow"] = dow
    cols["month"] = u64(rng.choice([2, 1 << 33, 1 << 62], n))  # DICT, 3 values
    cols["ras"] = rng.choice([60, 3600, 86400, -(1 << 31), (1 << 31) - 1], n).astype(np.int32)
    fin = 1790000000 + rng.integers(0, 7200, n)
    ext = rng.random(n)
    fin = np.where(ext < 0.05, -(1 << 63), np.where(ext > 0.95, (1 << 63) - 1, fin))  # FOR at width 64: RAW
    cols["finished_at"] = fin.astype(np.int64)
    cols["success"] = rng.integers(0, 5, n).astype(np.int32)
    cols["remedy_finished_at"] = np.where(rng.random(n) < 0.01, 1790000000 + rng.integers(0, 99, n), 0).astype(np.int64)
    cols["reset_interval"] = np.where(np.arange(n) < 3000, 7, rng.integers(-(1 << 31), (1 << 31) - 1, n)).astype(np.int32)
    return cols


def test_adversarial_blocks(am):
    """every block's mode is the documented rule's pick (all five occur), the packed blob decodes to the raw one and
    stays within the bound; ranges not a multiple of the block, one slot, ranges that start inside a word; a base past
    2^32; a restore of each packed blob checkpoints as the raw one"""
    rng = np.random.default_rng(3)
    n = 3 * 1024 + 517
    base = (1 << 32) + 77
    s = am.Sweep(capacity=n, shard_base=base)
    try:
        s.load_range(0, _adversarial_cols(am, rng, n))
        modes = set()
        for first, m in ((0, n), (37, n - 100), (1, 1), (n - 1, 1), (1029, 2 * 1024), (5, 0)):
            raw, packed = _both(am, s, first, m)
            for name, dt, j0, cnt, e in pf.directory(packed)[0]:
                v = np.frombuffer(raw, np.uint8)
                off = dict((a, o) for a, _, o, _ in pf.sections(np.frombuffer(raw[:128], "<u8"))[0])[name]
                esize = np.dtype(dt).itemsize
                vals = v[off + j0 * esize:off + (j0 + cnt) * esize].view(dt)
                want = pf.best_mode(vals, pf.NONE.get(name, 0))
                assert (e["mode"], e["width"], e["aux"]) == want[:3], (first, m, name, j0, e, want)
                modes.add(e["mode"])
            t = am.Sweep(capacity=n + 10, shard_base=base - 10)
            try:
                t.restore(packed)
                assert t.checkpoint(first + 10, m) == raw
            finally:
                t.close()
        assert modes == set(range(5)), modes
    finally:
        s.close()


def _set_entry(blob, b, **kw):
    out = bytearray(blob)
    e = np.frombuffer(bytes(out[128 + 16 * b:128 + 16 * b + 16]), pf.ENTRY).copy()
    for k, v in kw.items():
        e[0][k] = v
    out[128 + 16 * b:128 + 16 * b + 16] = e.tobytes()
    return bytes(out)


def _bad_dict_code(blob):
    """a DICT block whose dictionary is not a power of two long, with one code set past it"""
    blocks, pay = pf.directory(blob)
    for b, (name, dt, j0, cnt, e) in enumerate(blocks):
        if e["mode"] == pf.DICT and e["aux"] & (e["aux"] - 1):
            esize = np.dtype(dt).itemsize
            at = pay + e["off"] + (e["aux"] * esize + 7) // 8 * 8
            out = bytearray(blob)
            out[at] = (out[at] & ~((1 << e["width"]) - 1)) | ((1 << e["width"]) - 1)  # (code 0 := all ones)
            return bytes(out)
    raise AssertionError("no DICT block with a spare code")


def _refusals(am, packed, delta):
    """(what, blob, is a delta) of every malformed case"""
    out = []
    for what, blob, is_delta in (("full", packed, False), ("delta", delta, True)):
        blocks, pay = pf.directory(blob)
        nb = len(blocks)
        last = blocks[-1][4]
        for_b = next(b for b, x in enumerate(blocks) if x[4]["mode"] == pf.FOR and x[4]["width"] > 0)
        e = blocks[for_b][4]
        ver = bytearray(blob)
        ver[8] = 3
        cases = [("truncated", blob[:-8]), ("truncated directory", blob[:128 + 8]),
                 ("unknown version", bytes(ver)),
                 ("offset past the payload", _set_entry(blob, nb - 1, off=last["off"] + (1 << 40))),
                 ("offset not the previous end", _set_entry(blob, for_b, off=e["off"] + 8)),
                 ("width past 64", _set_entry(blob, for_b, width=65)),
                 ("width past the element", _set_entry(blob, 0, mode=pf.FOR, width=8 * np.dtype(blocks[0][1]).itemsize + 1)),
                 ("size that does not fit the mode", _set_entry(blob, for_b, width=e["width"] + 1)),
                 ("unknown mode", _set_entry(blob, for_b, mode=5)),
                 ("reserved word", _set_entry(blob, for_b, zero=1)),
                 ("DICT code past the dictionary", _bad_dict_code(blob)),
                 ("flipped payload byte", _flip(blob, pay + e["off"] + 8))]
        out += [(f"{what}: {c}", b, is_delta) for c, b in cases]
    return out


def test_refusals_change_nothing(am, zmap):
    """every malformed packed blob is refused (AM_E_INVAL) before anything changes: a standby with a call staged is
    byte for byte a twin that never saw the blob, and the refused call launched at most the decode and verify passes"""
    rng = np.random.default_rng(6)
    n, T = 4000, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    try:
        recs = _records(am, zmap, rng, n, T, True)
        recs["ras"] = rng.choice([60, 3600, 86400], n)  # (DICT blocks of 3 values)
        s.upsert(np.arange(n), recs)
        s.tick(T + 1)
        s.set_checkpoint_packing(True)
        root = s.checkpoint_chain(0, n)
        s.upsert(np.arange(0, n, 2), recs[:n // 2])
        s.post_result(rng.choice(n, 300), rng.integers(0, 3, 300).astype(np.uint8))
        s.tick(T + 2)
        delta, k = s.checkpoint_delta()
        assert k > 2048
        for what, blob, is_delta in _refusals(am, root, delta):
            pair = []
            for _ in range(2):
                sb = am.Sweep(capacity=n)
                sb.set_hold_in_flight(True)
                if is_delta:
                    sb.restore(root)
                sb.upsert([3], _junk(am, 1))  # (staged: a refusal drains nothing)
                pair.append(sb)
            try:
                c0 = pair[0].launch_count
                with pytest.raises(am.AmError) as e:
                    (pair[0].restore_delta if is_delta else pair[0].restore)(blob)
                assert e.value.code == am.AM_E_INVAL, (what, e.value.code)
                assert pair[0].launch_count - c0 <= 4, what  # (directory check, decode, verify passes: no drain)
                assert pair[0].checkpoint(0, n) == pair[1].checkpoint(0, n), what
                if "truncated" in what or "version" in what:  # (refused by the header checks alone)
                    with pytest.raises(am.AmError):
                        (am.checkpoint_delta_info if is_delta else am.checkpoint_info)(blob)
            finally:
                for sb in pair:
                    sb.close()
        sb = _standby(am, root, n, 0)  # (the blobs themselves apply)
        try:
            sb.restore_delta(delta)
            assert sb.checkpoint(0, n) == _full(s, 0, n, False)
        finally:
            sb.close()
    finally:
        s.close()


def test_nospace_after_the_encode(am, zmap):
    """a packed blob's AM_E_NOSPACE reports its packed length after the passes; a refused packed delta commits
    nothing"""
    rng = np.random.default_rng(2)
    n, T = 3000, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    try:
        s.set_checkpoint_packing(True)
        packed = s.checkpoint(0, n)
        need = ctypes.c_uint64(0)
        buf = np.zeros(len(packed) - 8, np.uint8)
        rc = s._lib.am_sweep_checkpoint(s._h, 0, n, buf.ctypes.data, len(buf), ctypes.byref(need))
        assert rc == am.AM_E_NOSPACE and need.value == len(packed)
        root = s.checkpoint_chain(0, n)
        sb = _standby(am, root, n, 0)
        s.post_result(np.arange(0, n, 3), np.full(len(range(0, n, 3)), 2, np.uint8))
        s.tick(T + 1)
        changed = ctypes.c_uint64(0)
        rc = s._lib.am_sweep_checkpoint_delta(s._h, buf.ctypes.data, 64, ctypes.byref(need), ctypes.byref(changed))
        assert rc == am.AM_E_NOSPACE and need.value > 64
        delta, k = s.checkpoint_delta()
        assert len(delta) == need.value and am.checkpoint_delta_info(delta)["seq"] == 1
        sb.restore_delta(delta)
        assert sb.checkpoint(0, n) == _full(s, 0, n, False)
        sb.close()
    finally:
        s.close()


def _launches(s, fn, *args):
    """the launches of one call into a buffer large enough (the wrappers retry after AM_E_NOSPACE)"""
    buf, need = np.zeros(1 << 22, np.uint8), ctypes.c_uint64(0)
    c0 = s.launch_count
    if fn == "am_sweep_checkpoint_delta":
        rc = s._lib.am_sweep_checkpoint_delta(s._h, buf.ctypes.data, len(buf), ctypes.byref(need),
                                              ctypes.byref(ctypes.c_uint64(0)))
    else:
        rc = getattr(s._lib, fn)(s._h, *args, buf.ctypes.data, len(buf), ctypes.byref(need))
    assert rc == 0
    return s.launch_count - c0, buf[:need.value].tobytes()


def test_launch_counts(am, zmap):
    rng = np.random.default_rng(8)
    n, T = 3000, T_PARIS
    s = _hold_handle(am, zmap, rng, n, T)
    try:
        assert _launches(s, "am_sweep_checkpoint", 0, n)[0] == 1  # (packing off: what it launched before)
        s.set_checkpoint_packing(True)
        c, packed = _launches(s, "am_sweep_checkpoint", 0, n)
        assert c == 4  # pack, sizes, scan, payloads
        assert _launches(s, "am_sweep_checkpoint", 0, 0)[0] == 0
        c, root = _launches(s, "am_sweep_checkpoint_chain", 0, n)
        assert c == 4
        sb = _standby(am, root, n, 0)
        s.tick(T + 1)
        c, d1 = _launches(s, "am_sweep_checkpoint_delta")
        k1 = am.checkpoint_delta_info(d1)["n_changed"]
        d1_launches = c
        assert k1 > 0 and d1_launches == 8  # diff, scan, compaction, pack, sizes, scan, payloads, commit
        b0 = sb.launch_count
        sb.restore_delta(d1)  # directory check, decode, offsets and sections verified, scatter, plane rebuild
        assert sb.launch_count - b0 == 6
        sb.close()
        t = _fresh(am, n, 0, am.checkpoint_info(packed))
        c0 = t.launch_count
        t.restore(packed)
        r = t.launch_count - c0
        t.close()
        t = _fresh(am, n, 0, am.checkpoint_info(packed))
        c0 = t.launch_count
        t.restore(pf.decode(packed))
        assert r - (t.launch_count - c0) == 2  # directory check and decode
        t.close()
    finally:
        s.close()


def test_full_size(am):
    """10 M config-5 records after a simulated hour with both holds and a tenth with workflow timeouts: a packed root
    and packed deltas after 1, 10 and 60 s, restored on a standby that then ticks bit-exact against the source"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import run_sim
    n, S = 10_000_000, 3600
    cols, sl, recs = run_sim.population(am, n, 3)
    src = am.Sweep(capacity=n)
    sb = None
    try:
        src.load_range(0, cols)
        src.set_hold_in_flight(True)
        src.set_hold_remedy(True)
        src.upsert(sl, recs)
        T = run_sim.amgen.T0_DAY_START
        src.simulate(T, S, BLOCKED, 3, run_sim.PARAMS)
        T += S
        src.set_checkpoint_packing(True)
        root = src.checkpoint_chain(0, n)
        info = am.checkpoint_info(root)
        assert info["version"] == 2 and info["bytes"] == len(root)
        sb = _fresh(am, n, 0, info)
        sb.restore(root)
        del root
        for period in (1, 10, 60):
            src.simulate(T, period, BLOCKED, 3, run_sim.PARAMS)
            T += period
            delta, k = src.checkpoint_delta()
            assert k > 0 and am.checkpoint_delta_info(delta)["version"] == 2
            sb.restore_delta(delta)
            del delta
        src.set_checkpoint_packing(False)
        assert sb.checkpoint(0, n) == src.checkpoint(0, n)
        for t in range(T, T + 3):
            ia, aa, sta = src.tick(t)
            ib, ab, stb = sb.tick(t)
            assert sta == stb and np.array_equal(ia, ib) and np.array_equal(aa, ab), t
    finally:
        src.close()
        if sb:
            sb.close()
