"""A sweep handle and its model (tests/handle_model.py), kept in step by every call.  After every tick the pair compares
everything the enabled switches expose: the list and statistics (except for tick_shard, whose list stays on the
device), the sixteen columns, am_sweep_in_flight and, with the remedy hold, am_sweep_remedy_in_flight, both timed-out
lists with the hold, am_sweep_last_changes and its columns with tracking, am_sweep_last_change_details with details."""
import os

import numpy as np
import pytest

import change_details_oracle
from handle_model import NO_TIMEOUTS, HandleModel, Refused, Tick


def emulated(am):
    return "emu" in os.path.basename(am.abi.LIB_PATH)


class DevOut:
    """output arrays of am_sweep_tick_device: torch device memory, or host memory on the CPU emulator"""

    def __init__(self, am, n):
        self.emu = emulated(am)
        self.n = n
        if self.emu:
            self.t = [np.zeros(n + 4, np.uint32), np.zeros(n + 4, np.uint8), np.zeros(4, np.uint32), np.zeros(16, np.uint64)]
            self.ptr = [a.ctypes.data for a in self.t]
        else:
            import torch
            self.t = [torch.zeros(n + 4, dtype=torch.int32, device="cuda"), torch.zeros(n + 4, dtype=torch.uint8, device="cuda"),
                      torch.zeros(4, dtype=torch.int32, device="cuda"), torch.zeros(16, dtype=torch.int64, device="cuda")]
            self.ptr = [a.data_ptr() for a in self.t]

    def tick(self, am, s, T, mode, cap=None, stream=None):
        cap = self.n if cap is None else cap
        s.tick_device(T, mode, self.ptr[0], self.ptr[1], cap, self.ptr[2], self.ptr[3],
                      stream=s.stream if stream is None else stream)
        if self.emu:
            idx, act, cnt, st = self.t
        else:
            import torch
            torch.cuda.synchronize()
            idx, act, cnt, st = [a.cpu().numpy() for a in self.t]
        k = int(cnt.view(np.uint32)[0])
        stats = dict(zip(am.abi.STAT_FIELDS, [int(v) for v in st.view(np.uint64)]))
        return idx.view(np.uint32)[:k].astype(np.uint64) + np.uint64(s.shard_base), act[:k].astype(np.uint32), stats


def check_changes(s, want, ocols, where, names=None):
    """the handle's changed set against the model's, its columns against the model's columns"""
    idx, cols = s.last_changes(names=names)
    np.testing.assert_array_equal(idx, want, err_msg=f"{where}: changed set")
    loc = (want - np.uint64(s.shard_base)).astype(np.int64)
    for name, a in cols.items():
        np.testing.assert_array_equal(a, ocols[name][loc], err_msg=f"{where}: {name}")
    return len(idx)


def check_details(s, want_idx, want, where):
    idx, det = s.last_change_details()
    np.testing.assert_array_equal(idx, want_idx, err_msg=f"{where}: listed slots")
    for name in change_details_oracle.DETAIL.names:
        np.testing.assert_array_equal(det[name], want[name], err_msg=f"{where}: {name}")
    return len(idx)


class Pair:
    """`n_or_cols`: the capacity, or columns to load into slots 0.. of a handle of their size.  `entry` is the tick
    entry point (tick, tick_short with `cap` entries and the rest paged, tick_view, tick_device or tick_shard).
    `every_slot` compares all columns of every swept slot; otherwise flags everywhere and the other columns of live
    slots (a slot removed in the drain of its upsert keeps different stale columns on the two sides)."""

    def __init__(self, am, zmap, n_or_cols, hold=False, remedy=False, track=False, details=False, entry="tick",
                 shard_base=0, seed=0, cap=1, every_slot=True):
        cols = None if isinstance(n_or_cols, int) else n_or_cols
        self.n = n_or_cols if cols is None else len(cols["flags"])
        self.am, self.entry, self.cap, self.every_slot = am, entry, cap, every_slot
        self.s = am.Sweep(capacity=self.n, shard_base=shard_base)
        self.m = HandleModel(zmap, self.n, shard_base, seed=seed)
        if seed:
            self.s.set_seed(seed)
        for on, switch in ((hold, self.set_hold), (remedy, self.set_remedy), (track, self.set_track),
                           (details, self.set_details)):
            if on:
                switch(True)
        if cols is not None:
            self.load(0, cols)
        self.dev = None
        self.timed_total = self.rtimed_total = self.started = self.listed = self.detailed = 0

    def close(self):
        self.s.close()

    # ---- calls, on both sides ----
    def upsert(self, slots, recs):
        self.s.upsert(slots, recs)
        self.m.upsert(slots, recs)

    def remove(self, slots):
        self.s.remove(slots)
        self.m.remove(slots)

    def post(self, slots, phase, rphase=None):
        self.s.post_result(slots, phase, rphase)
        self.m.post(slots, phase, rphase)

    def load(self, first, cols):
        self.s.load_range(first, cols)
        self.m.load(first, cols)

    def read(self, slots):
        self.s.read(slots)
        self.m.read(slots)

    def _switch(self, handle_call, model_call, on):
        """a switch on both sides; a refusal must be the same on both and is raised as the model's"""
        try:
            model_call(on)
        except Refused as r:
            with pytest.raises(self.am.AmError) as e:
                handle_call(on)
            assert e.value.code == r.code, (e.value.code, r.code)
            raise
        handle_call(on)

    def set_hold(self, on):
        self._switch(self.s.set_hold_in_flight, self.m.set_hold, on)

    def set_remedy(self, on):
        self._switch(self.s.set_hold_remedy, self.m.set_remedy, on)

    def set_track(self, on):
        self._switch(self.s.set_track_changes, self.m.set_track, on)

    def set_details(self, on):
        self._switch(self.s.set_change_details, self.m.set_details, on)

    # ---- queries: the handle's answers ----
    def in_flight(self):
        return self.s.in_flight(0, self.n)

    def remedy_in_flight(self):
        return self.s.remedy_in_flight(0, self.n)

    def cols(self):
        return self.s.read_range(0, self.n)

    def changes(self):
        return self.m.changes()

    def details(self):
        return self.m.details()

    # ---- the tick ----
    def _call(self, entry, T, mode, want):
        am, s = self.am, self.s
        if entry == "tick":
            return s.tick(T, mode=mode)
        if entry == "tick_short":
            try:
                return s.tick(T, mode=mode, cap=self.cap)
            except am.AmError as e:
                assert e.code == am.AM_E_NOSPACE
                idx, act, left = s.last_list(0, e.needed)
                assert left == e.needed == want.stats["n_emitted"]
                return idx, act, want.stats  # (an AM_E_NOSPACE tick: the statistics are not returned)
        if entry == "tick_view":
            i, a, st = s.tick_view(T, mode=mode)
            return i.astype(np.uint64) + np.uint64(s.shard_base), a.astype(np.uint32), st
        if entry == "tick_device":
            self.dev = self.dev or DevOut(am, self.n)
            return self.dev.tick(am, s, T, mode)
        s.tick_shard(T, mode=mode)
        return None

    def tick(self, T, mode=0, entry=None):
        """the model's tick, then the handle's through `entry`, then every comparison; the handle's answer in the
        model's shape (the model's list for tick_shard)"""
        am, s, m = self.am, self.s, self.m
        entry = entry or self.entry
        what = (entry, mode, T)
        before = m.rsince.copy()
        want = m.tick(T, mode)
        self.started += int(((m.rsince == T) & (before != T)).sum())
        got = self._call(entry, T, mode, want)
        h = m.hwm
        dev = s.read_range(0, h)
        ocols = {k: v[:h] for k, v in m.cols().items()}
        if got is None:
            got = want[:3]
        else:
            gi, ga, gs = got
            assert gs == want.stats, (what, {k: (gs[k], want.stats[k]) for k in gs if gs[k] != want.stats[k]})
            np.testing.assert_array_equal(gi, want.idx, err_msg=f"{what}: idx")
            np.testing.assert_array_equal(ga, want.act, err_msg=f"{what}: act")
        if self.every_slot:
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], ocols[name], err_msg=f"{what} {name}")
        else:
            live = m.live(np.arange(h))
            for name in am.COLUMN_NAMES:
                keep = live | (name == "flags")
                np.testing.assert_array_equal(dev[name][keep], ocols[name][keep], err_msg=f"{what} {name}")
        timed = rtimed = NO_TIMEOUTS
        if m.hold:
            np.testing.assert_array_equal(s.in_flight(0, self.n), m.in_flight(), err_msg=str(what))
            timed, rtimed = s.last_timed_out(), s.last_remedy_timed_out()
            for k in range(2):
                np.testing.assert_array_equal(timed[k], want.timed_out[k], err_msg=str(what))
                np.testing.assert_array_equal(rtimed[k], want.remedy_timed_out[k], err_msg=str(what))
            self.timed_total += len(timed[0])
            self.rtimed_total += len(rtimed[0])
        if m.remedy:
            np.testing.assert_array_equal(s.remedy_in_flight(0, self.n), m.remedy_in_flight(), err_msg=str(what))
        if m.track:
            self.listed += check_changes(s, m.changes(), m.cols(), what)
        if m.details_on:
            self.detailed += check_details(s, m.changes(), m.details(), what)
        return Tick(got[0], got[1], got[2], timed, rtimed)
