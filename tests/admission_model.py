"""tests/handle_model.py's HandleModel with a submit budget (am_sweep_set_submit_budget): the budget, the admission
state (allocated at the first finite budget, like the handle's) and per slot the second since which it waits for
admission.  The tick is tests/admission_oracle.py around the model's own tick; the waits end at a remove, a load, a
posted workflow phase and when the hold is toggled (which also makes the budget unlimited); an upsert keeps them."""
import numpy as np

import admission_oracle as ao
from handle_model import E_INVAL, HandleModel, Refused, Tick


class AdmissionModel(HandleModel):
    def __init__(self, zmap, capacity, shard_base=0, seed=0, **switches):
        self.budget = ao.UNLIMITED
        self.adm = False  # the admission state exists
        self.wait = np.full(capacity, ao.NOT_WAITING, dtype=np.int64)
        self.admission = ao.empty_admission()
        self._admit = False
        super().__init__(zmap, capacity, shard_base, seed, **switches)

    def admitting(self):
        return self.adm and self.hold

    # ---- calls ----
    def set_budget(self, per_tick):
        if not self.hold:
            raise Refused(E_INVAL)
        v = ao.UNLIMITED if per_tick is None else int(per_tick)
        if v != ao.UNLIMITED:
            self.adm = True
        self.budget = v

    def set_hold(self, on):
        if bool(on) != self.hold:
            self.budget = ao.UNLIMITED
            self.wait[:] = ao.NOT_WAITING
            self.admission = ao.empty_admission()
        super().set_hold(on)

    def remove(self, idx):
        super().remove(idx)
        self.wait[np.asarray(idx, dtype=np.int64)] = ao.NOT_WAITING

    def post(self, idx, phase, rphase=None):
        super().post(idx, phase, rphase)
        idx = np.asarray(idx, dtype=np.int64)
        self.wait[idx[np.asarray(phase) != 0]] = ao.NOT_WAITING

    def load(self, first, cols):
        super().load(first, cols)
        self.wait[first:first + len(cols["flags"])] = ao.NOT_WAITING

    # ---- the tick ----
    def tick(self, T, mode=0):
        self._admit = self.admitting()
        try:
            return super().tick(T, mode)
        finally:
            self._admit = False

    def _sweep(self, cols, runs, T, P, mode, seed):
        if not self._admit:
            return super()._sweep(cols, runs, T, P, mode, seed)
        h = len(cols["flags"])
        wait = self.wait[:h]
        force = np.flatnonzero((wait != ao.NOT_WAITING) & ao.can_be_due(cols["flags"]) & ~self.held())
        forced = ao.force_due(cols, force)
        try:
            out = super()._sweep(cols, runs, T, P, mode, seed)
        finally:
            ao.restore(cols, forced)
        since, deadline = runs[0], runs[1]
        idx, act, st, self.admission = ao.cut(out.idx, out.act, out.stats, wait, since, deadline, self.budget, T,
                                              self.shard_base)
        return Tick(idx, act, st, out.timed_out, out.remedy_timed_out)

    # ---- queries ----
    def deferred(self, first=0, n=None, idx=None):
        sl = self._slots(first, n, idx)
        return self.wait[sl].copy()

    def last_admission(self):
        if not self.adm:
            raise Refused(E_INVAL)
        return dict(self.admission)
