"""tests/admission_model.py's AdmissionModel (tests/handle_model.py's HandleModel with a submit budget) with spec updates
(am_sweep_update_spec, DESIGN §6 item 20).

update_spec of a live slot takes the masks, ras, runs_limit, reset_interval, W and the spec bits of flags (the latest
entry of a slot wins) and changes nothing else: not the counters, the finish times, the pending, remedy and timer bits,
since, the deadlines, the waits for admission or the starts the details take at the posts.  One of a tombstone changes
nothing.  The handle applies only a slot's latest spec update of a drain, on the flags the drain found:
STOPPED_REPORTED stays iff it was set there, that kind was STOPPED and the new kind is.  So the model keeps, per slot,
the flags before its first spec update since the last drain (an upsert, remove or load of the slot drops them);
drained() forgets them.  Every call of the model that drains on the handle (a tick, run_ticks, a load, a read, turning
details on) calls it, and a driver calls it for the handle's queries and checkpoints."""
import numpy as np

from admission_model import AdmissionModel

KIND_MASK, KIND_STOPPED = 0x7, 1
F_TOMBSTONE, F_STOPPED_REPORTED = 1 << 8, 1 << 9
F_SPEC_MASK = KIND_MASK | 1 << 3 | 0xFF << 16 | 0xFF << 24  # AM_F_SPEC_MASK: kind, HAS_REMEDY, fail-p, zone
SPEC_COLUMNS = ("minute", "hour", "dom", "month", "dow", "ras", "runs_limit", "reset_interval")


def _last_of(idx):
    """positions of the last occurrence of every distinct slot of idx (a later entry of a call wins)"""
    _, rev = np.unique(idx[::-1], return_index=True)
    return len(idx) - 1 - rev


class SpecModel(AdmissionModel):
    def __init__(self, zmap, capacity, shard_base=0, seed=0, **switches):
        self.spec_base = np.full(capacity, -1, dtype=np.int64)  # -1: no spec update since the last drain
        super().__init__(zmap, capacity, shard_base, seed, **switches)

    def drained(self):
        self.spec_base[:] = -1

    def _drop(self, slots):
        super()._drop(slots)
        self.spec_base[np.asarray(slots, dtype=np.int64)] = -1

    # ---- calls ----
    def update_spec(self, idx, recs):
        idx = np.asarray(idx, dtype=np.int64)
        last = _last_of(idx)
        sl, r = idx[last], last
        live = (self.c["flags"][sl] & np.uint32(F_TOMBSTONE)) == 0
        sl, r = sl[live], r[live]
        f, g = self.c["flags"][sl], np.asarray(recs["flags"][r], dtype=np.uint32)
        first = self.spec_base[sl] < 0
        self.spec_base[sl[first]] = f[first]
        base = self.spec_base[sl].astype(np.uint32)
        for name in SPEC_COLUMNS:
            self.c[name][sl] = recs[name][r]
        nf = (f & np.uint32(~(F_SPEC_MASK | F_STOPPED_REPORTED) & 0xFFFFFFFF)) | (g & np.uint32(F_SPEC_MASK))
        stays = ((base & np.uint32(KIND_MASK)) == KIND_STOPPED) & ((g & np.uint32(KIND_MASK)) == KIND_STOPPED)
        self.c["flags"][sl] = nf | np.where(stays, base & np.uint32(F_STOPPED_REPORTED), np.uint32(0))
        self.wf[sl] = recs["wf_timeout"][r]

    # ---- the calls that drain on the handle ----
    def load(self, first, cols):
        self.drained()
        super().load(first, cols)

    def read(self, slots=None):
        self.drained()
        super().read(slots)

    def set_details(self, on):
        turning_on = bool(on) and not self.details_on
        super().set_details(on)  # (refused while tracking is off: the handle drains nothing then)
        if turning_on:
            self.drained()

    def tick(self, T, mode=0):
        out = super().tick(T, mode)  # (a refused tick drains nothing)
        self.drained()
        return out

    def run_ticks(self, T0, n, mode=0, seed=0):
        rows = super().run_ticks(T0, n, mode, seed)
        self.drained()
        return rows
