"""GPU parity tests: the CUDA sweep, called through the C-ABI, against the CPU
oracle on the same seeded inputs — bit-exact due lists, action bytes, statistics
and every mutated status column (SURVEY.md §8c/§8d).

Bit-exact here means: against our restatement of hcc.go + robfig/cron v3.0.1;
the Go binary could not be executed in this environment (oracle/amsweep_oracle.h).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T0 = 1789982100      # 2026-09-21 09:15:00 UTC Monday
T_OCT1 = 1790812800  # 2026-10-01 00:00:00 UTC Thursday


def _gen_pair(gen, am, orc, config, seed, n, T, first=0):
    """Columns through the PRODUCT classifier and through the ORACLE classifier."""
    prod = gen.fill(config, seed, first, n, T, am.load().am_healthcheck_classify)
    orac = gen.fill(config, seed, first, n, T, orc.load().orc_classify)
    for name in am.COLUMN_NAMES:  # upsert-time parity (parser + ladder)
        np.testing.assert_array_equal(prod[name], orac[name], err_msg=f"classify column {name}")
    return prod, orac


def _assert_tick_equal(am, got, want, sweep, ocols, n, what=""):
    gi, ga, gs = got
    wi, wa, ws = want
    assert gs == ws, f"{what}: stats differ\n gpu={gs}\n cpu={ws}"
    np.testing.assert_array_equal(gi, wi, err_msg=f"{what}: due indices")
    np.testing.assert_array_equal(ga, wa, err_msg=f"{what}: action bytes")
    dev = sweep.read_range(0, n)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(dev[name], ocols[name], err_msg=f"{what}: column {name}")


@pytest.mark.parametrize("config,n", [(1, 1000), (11, 1000)])
def test_config1_interval_1000(am, orc, gen, config, n):
    """BASELINE configs[0]: 1 000 checks, repeatAfterSec=60 / "@every 1m" — same due-set."""
    prod, orac = _gen_pair(gen, am, orc, config, 1, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        got = s.tick(T0)
        want = orc.sweep(orac, T0)
        _assert_tick_equal(am, got, want, s, orac, n, f"config {config}")
        assert 0.35 * n < got[2]["n_submit_hc"] < 0.65 * n  # ~50 % due by construction
    # both variants of inlineHello.yaml yield the identical due-set
    a = gen.fill(1, 1, 0, n, T0, am.load().am_healthcheck_classify)
    b = gen.fill(11, 1, 0, n, T0, am.load().am_healthcheck_classify)
    with am.Sweep(capacity=n) as sa, am.Sweep(capacity=n) as sb:
        sa.load_range(0, a)
        sb.load_range(0, b)
        ia, _, _ = sa.tick(T0)
        ib, _, _ = sb.tick(T0)
        np.testing.assert_array_equal(ia, ib)


@pytest.mark.parametrize("T", [T0, T_OCT1, T0 + 1, T0 + 45, 1767225600, 1709164800])
@pytest.mark.parametrize("n", [1, 63, 1024, 1025, 200_003])
def test_config2_mixed(am, orc, gen, T, n):
    """BASELINE configs[1] population at oracle-friendly sizes, several ticks, ragged sizes."""
    prod, orac = _gen_pair(gen, am, orc, 2, 2, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        got = s.tick(T)
        want = orc.sweep(orac, T)
        _assert_tick_equal(am, got, want, s, orac, n, f"config2 n={n} T={T}")
        # second tick one second later: STOPPED is reported once only
        got2 = s.tick(T + 1)
        want2 = orc.sweep(orac, T + 1)
        _assert_tick_equal(am, got2, want2, s, orac, n, "config2 second tick")


@pytest.mark.parametrize("T", [T0, T_OCT1, T0 + 1])
@pytest.mark.parametrize("n", [1000, 300_007])
def test_config3_remedy_state_machine(am, orc, gen, T, n):
    """BASELINE configs[2]: 50 % pending Failed, 25 % Succeeded; remedy gate and counters.
    T0 + 1 is off the minute: the no-masks kernel variant takes the dense result path too."""
    prod, orac = _gen_pair(gen, am, orc, 3, 3, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        got = s.tick(T)
        want = orc.sweep(orac, T)
        _assert_tick_equal(am, got, want, s, orac, n, f"config3 n={n}")
        st = got[2]
        if n > 100_000 and T == T0:  # remedyFinishedAt is within 600 s of T0: skips only there
            for k in ("n_run_remedy", "n_remedy_skip", "n_reset_on_pass", "n_reset_on_interval",
                      "n_anomaly", "n_result_ok", "n_result_fail", "n_remedy_ok", "n_remedy_fail"):
                assert st[k] > 0, f"population does not exercise {k}"


def test_full_scan_mode_equals_default(am, orc, gen):
    n = 50_000
    prod, orac = _gen_pair(gen, am, orc, 2, 7, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        for T in (T0 + 7, T0 + 60):
            got = s.tick(T, mode=am.SWEEP_FULL_SCAN)
            want = orc.sweep(orac, T)
            _assert_tick_equal(am, got, want, s, orac, n, f"full-scan T={T}")


def test_remedy_gate_known_answers(am, orc):
    """SURVEY Appendix C remedy vectors, through upsert + post_result + tick."""
    T = T0
    A = am
    rows = [  # runsLimit, resetInterval, RT, d (None = nil), expected action bits
        (2, 300, 1, 10, A.ACT_RUN_REMEDY),
        (2, 300, 2, 300, A.ACT_REMEDY_SKIP),
        (2, 300, 2, 301, A.ACT_RESET_ON_INTERVAL | A.ACT_RUN_REMEDY),
        (0, 300, 9, 10, A.ACT_RUN_REMEDY),
        (2, 0, 9, 10, A.ACT_RUN_REMEDY),
        (2, 300, 2, None, A.ACT_ANOMALY),
    ]
    recs = np.zeros(len(rows) + 2, dtype=am.RECORD_DTYPE)
    for k, (lim, rst, rt, d, _) in enumerate(rows):
        rc, r = am.classify(repeat_after_sec=3600, has_remedy=True, remedy_runs_limit=lim,
                            remedy_reset_interval=rst, remedy_total_runs=rt,
                            remedy_failed_count=rt, finished_at=T - 5,
                            remedy_finished_at=None if d is None else T - d)
        assert rc == 0
        recs[k] = r[0]
    # pending Succeeded with RT>=1 resets; with RT==0 leaves everything alone
    for k, rt in ((len(rows), 3), (len(rows) + 1, 0)):
        rc, r = am.classify(repeat_after_sec=3600, has_remedy=True, remedy_total_runs=rt,
                            remedy_success_count=rt, finished_at=T - 5,
                            remedy_finished_at=(T - 50) if rt else None)
        recs[k] = r[0]
    n = len(recs)
    with am.Sweep(capacity=n) as s:
        s.upsert(np.arange(n), recs)
        phase = np.array([am.PHASE_FAILED] * len(rows) + [am.PHASE_SUCCEEDED] * 2, dtype=np.uint8)
        rphase = np.array([am.PHASE_SUCCEEDED] * n, dtype=np.uint8)
        s.post_result(np.arange(n), phase, rphase)
        idx, act, st = s.tick(T)
        got = dict(zip(idx.tolist(), act.tolist()))
        for k, row in enumerate(rows):
            assert got.get(k, 0) == row[4], f"row {k}: {row} -> {got.get(k, 0):#x}"
        assert got.get(len(rows)) == A.ACT_RESET_ON_PASS
        assert len(rows) + 1 not in got
        after = s.read(np.arange(n))
        assert after["remedy_total"][0] == 2 and after["remedy_success"][0] == 1
        assert after["remedy_total"][2] == 1          # reset then one run
        assert after["remedy_total"][1] == 2          # skipped: untouched
        assert after["remedy_total"][len(rows)] == 0 and after["remedy_finished_at"][len(rows)] == 0
        assert (after["finished_at"] == T).all()      # every record took a result
        assert (after["flags"] & (A.F_PENDING_OK | A.F_PENDING_FAIL | A.F_REMEDY_PENDING)).max() == 0
        # oracle agrees record by record
        oc = am.records_to_columns(recs)
        bits = np.where(phase == am.PHASE_FAILED, A.F_PENDING_FAIL, A.F_PENDING_OK).astype(np.uint32)
        oc["flags"] = oc["flags"] | bits | np.uint32(A.F_REMEDY_PENDING | A.F_REMEDY_OUTCOME_OK)
        wi, wa, ws = orc.sweep(oc, T)
        np.testing.assert_array_equal(idx, wi)
        np.testing.assert_array_equal(act, wa)
        assert st == ws
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(after[name], oc[name], err_msg=name)


def test_upsert_remove_and_deferred_remedy_result(am, orc, gen):
    n = 5000
    prod, orac = _gen_pair(gen, am, orc, 3, 11, n, T0)
    recs = am.columns_to_records(prod)
    with am.Sweep(capacity=n + 100) as s:
        # scatter in a shuffled order, in two batches, as Reconcile workers would
        perm = np.random.default_rng(0).permutation(n)
        s.upsert(perm[: n // 2], recs[perm[: n // 2]])
        s.upsert(perm[n // 2:], recs[perm[n // 2:]])
        gone = np.array([3, 77, 1024, n - 1], dtype=np.uint64)
        s.remove(gone)
        orac["flags"][gone.astype(np.int64)] = am.F_TOMBSTONE
        got = s.tick(T0)
        assert s.size == n
        want = orc.sweep(orac, T0)
        dev = s.read_range(0, n)
        assert got[2] == want[2]
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
        for name in am.COLUMN_NAMES:
            keep = np.ones(n, bool)
            keep[gone.astype(np.int64)] = False  # tombstoned slots keep only the flag
            np.testing.assert_array_equal(dev[name][keep], orac[name][keep], err_msg=name)
        assert (dev["flags"][gone.astype(np.int64)] == am.F_TOMBSTONE).all()
        # a remedy that finishes on its own (hcc.go:821-851), posted later
        live = np.flatnonzero((orac["flags"] & 7 == am.KIND_INTERVAL) & (orac["flags"] & am.F_TOMBSTONE == 0))[:50]
        s.post_result(live, np.zeros(len(live), np.uint8), np.full(len(live), am.PHASE_FAILED, np.uint8))
        orac["flags"][live] |= am.F_REMEDY_PENDING
        got = s.tick(T0 + 3)
        want = orc.sweep(orac, T0 + 3)
        assert got[2] == want[2] and got[2]["n_remedy_fail"] == len(live)
        dev = s.read(live)
        np.testing.assert_array_equal(dev["remedy_failed"], orac["remedy_failed"][live])
        np.testing.assert_array_equal(dev["remedy_finished_at"], np.full(len(live), T0 + 3))


def test_nospace_reports_needed_size(am, gen):
    n = 4096
    prod = gen.fill(1, 1, 0, n, T0, am.load().am_healthcheck_classify)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        with pytest.raises(am.AmError) as ei:
            s.tick(T0, cap=10)
        assert ei.value.code == am.AM_E_NOSPACE
        full_idx, _, st = s.tick(T0)
        assert ei.value.needed == st["n_emitted"] == len(full_idx)
        np.testing.assert_array_equal(ei.value.partial[0], full_idx[:10])


def test_shard_base_gives_global_indices(am, orc, gen):
    n, base = 3000, 12_500_000
    prod = gen.fill(2, 4, base, n, T0, am.load().am_healthcheck_classify)
    orac = gen.fill(2, 4, base, n, T0, orc.load().orc_classify)
    with am.Sweep(capacity=n, shard_base=base) as s:
        s.load_range(0, prod)
        got = s.tick(T0)
        want = orc.sweep(orac, T0, shard_base=base)
        assert got[2] == want[2]
        np.testing.assert_array_equal(got[0], want[0])
        assert got[0].min() >= base


def test_closed_loop_many_ticks(am, orc, gen):
    """BASELINE configs[4] in miniature: consecutive ticks, due records complete at once."""
    n, seed = 20_000, 5
    for config in (5, 55):
        prod, orac = _gen_pair(gen, am, orc, config, seed, n, T0)
        with am.Sweep(capacity=n) as s:
            s.load_range(0, prod)
            s.set_seed(seed)
            for k in range(0, 130):
                T = T0 - 60 + k  # crosses two minute boundaries
                got = s.tick(T, mode=am.SWEEP_CLOSED_LOOP)
                want = orc.sweep(orac, T, mode=1, seed=seed)
                assert got[2] == want[2], f"config {config} tick {k}"
                np.testing.assert_array_equal(got[0], want[0])
                np.testing.assert_array_equal(got[1], want[1])
            dev = s.read_range(0, n)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], orac[name], err_msg=f"config {config} {name}")


def test_run_ticks_streaming_matches_single_ticks(am, orc, gen):
    n, seed, nt = 30_000, 9, 200
    prod, orac = _gen_pair(gen, am, orc, 5, seed, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        stats = s.run_ticks(T0 - 30, nt, mode=am.SWEEP_CLOSED_LOOP, seed=seed)
        assert s.last_kernel_ms > 0
        for k in range(nt):
            _, _, ws = orc.sweep(orac, T0 - 30 + k, mode=1, seed=seed)
            gs = {f: int(stats[f][k]) for f in am.abi.STAT_FIELDS}
            assert gs == ws, f"tick {k}"
        dev = s.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], orac[name], err_msg=name)


def _post_results(am, sweeps, ocols, n, density, seed):
    """Workflow phases and remedy phases posted by separate calls (the reference's two watch loops) on
    every `step`-th slot of each handle; the oracle's columns get the same pending bits.  Every 23rd slot
    stays at most an eighth of the records in staged results (the drain's sparse path,
    apply_results_now_kernel); every second slot is the dense path (apply_result_ops_kernel)."""
    rng = np.random.default_rng(seed)
    slots = np.arange(int(rng.integers(0, 23)), n, 23 if density.startswith("sparse") else 2)
    phase = rng.integers(1, 3, len(slots)).astype(np.uint8)
    rphase = rng.integers(0, 3, len(slots)).astype(np.uint8)
    for s in sweeps:
        s.post_result(slots, phase)
        s.post_result(slots, np.zeros_like(phase), rphase)
    hc = np.uint32(am.F_PENDING_OK | am.F_PENDING_FAIL)
    rm = np.uint32(am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK)
    f = ocols["flags"][slots]
    f = (f & ~hc) | np.where(phase == am.PHASE_SUCCEEDED, am.F_PENDING_OK, am.F_PENDING_FAIL).astype(np.uint32)
    rbits = np.where(rphase == am.PHASE_SUCCEEDED, rm, np.uint32(am.F_REMEDY_PENDING)).astype(np.uint32)
    f = np.where(rphase != 0, (f & ~rm) | rbits, f)
    ocols["flags"][slots] = f
    return slots


RUN_TICKS_CASES = [
    (5, True, -30, 200, 0, None),      # config-2 mix (cron + intervals), closed loop, three minute boundaries
    (22, False, -70, 150, 0, None),    # open loop, zone-bound schedules among the crons
    (55, True, -75, 160, 7, None),     # remedy mix, closed loop, short blocks
    (3, False, -10, 90, 0, None),      # open loop: posted results and remedy gates at the first tick, then unarmed checks every tick
    (2, False, 45, 70, 64, None),      # open loop config 2
    (5, True, -100, 300, 128, None),   # the longest blocks
    (5, True, 0, 1, 0, None),          # a single tick
    # results posted through the C-ABI just before the run: applied by the run's first tick
    (3, False, 0, 3, 0, "sparse"),
    (3, True, -10, 90, 7, "sparse"),
    (55, False, -75, 160, 1, "sparse"),
    (3, False, 0, 3, 0, "dense"),
    (55, True, -10, 150, 128, "dense"),
    (3, False, 0, 3, 0, "sparse-late"),  # AMSWEEP_EARLY_RESULTS=0: every result applied inside the sweep
    (5, True, -30, 200, 96, "sparse-late"),
]


# (the cases without posted results keep the ids they had before the `posted` column existed)
@pytest.mark.parametrize("config,closed,start,nt,block,posted", RUN_TICKS_CASES,
                         ids=["-".join(str(v) for v in case if v is not None) for case in RUN_TICKS_CASES])
def test_run_ticks_blocked_equals_the_oracle_tick_by_tick(am, orc, gen, monkeypatch, config, closed, start, nt, block, posted):
    """AM_SWEEP_BLOCKED: up to 64 ticks per pass over the columns, every record stepped from event to event
    in registers (sweep_block.cuh).  Per-tick statistics — counts, action counts, index checksums, result
    counters — and every column afterwards must equal the oracle's tick-by-tick evaluation, and the
    library's own unblocked run; so must the host tick that follows the run."""
    n, seed = 30_000, 9
    if block:
        monkeypatch.setenv("AMSWEEP_BLOCK_TICKS", str(block))
    if posted == "sparse-late":
        monkeypatch.setenv("AMSWEEP_EARLY_RESULTS", "0")
    prod, orac = _gen_pair(gen, am, orc, config, seed, n, T0)
    mode = am.SWEEP_CLOSED_LOOP if closed else 0
    with am.Sweep(capacity=n) as s, am.Sweep(capacity=n) as s1:
        s.load_range(0, prod)
        s1.load_range(0, prod)
        if posted:
            _post_results(am, (s, s1), orac, n, posted, seed)
        l0 = s.launch_count
        stats = s.run_ticks(T0 + start, nt, mode=mode | am.SWEEP_BLOCKED, seed=seed)
        drain = 3 if posted else 0  # mark, apply, clear the staged results
        assert s.launch_count - l0 <= (nt + (block or 96) - 1) // (block or 96) + 2 + drain  # one launch per block (+ a zone-window split)
        plain = s1.run_ticks(T0 + start, nt, mode=mode, seed=seed)
        emitted = 0
        for k in range(nt):
            _, _, ws = orc.sweep(orac, T0 + start + k, mode=mode, seed=seed)
            gs = {f: int(stats[f][k]) for f in am.abi.STAT_FIELDS}
            assert gs == ws, f"tick {k}: blocked {gs} oracle {ws}"
            assert gs == {f: int(plain[f][k]) for f in am.abi.STAT_FIELDS}, f"tick {k} vs unblocked"
            emitted += ws["n_emitted"]
        assert emitted > nt
        dev = s.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], orac[name], err_msg=name)
        # the next host tick continues from where the run left off, on both handles
        T = T0 + start + nt
        s.set_seed(seed)
        s1.set_seed(seed)
        want = orc.sweep(orac, T, mode=mode, seed=seed)
        _assert_tick_equal(am, s.tick(T, mode=mode), want, s, orac, n, "tick after the blocked run")
        got = s1.tick(T, mode=mode)
        assert got[2] == want[2], "tick after the unblocked run"
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])


@pytest.mark.parametrize("consumer", ["tick", "tick_view", "tick_device", "next_due", "repeat_after_sec", "read"])
@pytest.mark.parametrize("density", ["sparse", "dense", "sparse-late"])
def test_posted_results_then_any_consumer_then_a_tick(am, orc, gen, monkeypatch, density, consumer):
    """Results posted through the C-ABI (phases by separate calls, sparse / dense / sparse with the early
    path off), then ONE call that drains them — a host tick, a tick view, a device tick, next_due,
    repeat_after_sec or a read — then a host tick.  Both must equal the oracle.  (The runs of ticks as
    consumers: test_run_ticks_blocked_equals_the_oracle_tick_by_tick.)"""
    import ctypes as C
    n, seed = 40_000, 3
    if density == "sparse-late":
        monkeypatch.setenv("AMSWEEP_EARLY_RESULTS", "0")
    prod, orac = _gen_pair(gen, am, orc, 3, seed, n, T0)
    T = T0
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        slots = _post_results(am, (s,), orac, n, density, seed)
        ticked = consumer.startswith("tick")
        if consumer == "tick":
            _assert_tick_equal(am, s.tick(T), orc.sweep(orac, T), s, orac, n, "tick")
        elif consumer == "tick_view":
            vi, va, st = s.tick_view(T)
            wi, wa, ws = orc.sweep(orac, T)
            assert st == ws
            np.testing.assert_array_equal(vi.astype(np.uint64), wi)
            np.testing.assert_array_equal(va.astype(np.uint32), wa)
        elif consumer == "tick_device":
            import torch
            dev = torch.device("cuda:0")
            d_idx = torch.empty(n, dtype=torch.int32, device=dev)
            d_act = torch.empty(n, dtype=torch.uint8, device=dev)
            d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
            d_st = torch.zeros(16, dtype=torch.int64, device=dev)
            stream = torch.cuda.current_stream()
            s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            wi, wa, ws = orc.sweep(orac, T)
            cnt = int(d_cnt.item())
            assert cnt == len(wi)
            np.testing.assert_array_equal(d_idx[:cnt].cpu().numpy().astype(np.uint64), wi)
            np.testing.assert_array_equal(d_act[:cnt].cpu().numpy().astype(np.uint32), wa)
            assert dict(zip(am.abi.STAT_FIELDS, [int(v) & ((1 << 64) - 1) for v in d_st.cpu().tolist()])) == ws
        elif consumer == "next_due":
            assert s.next_due(T) == T + 1  # results are waiting
        elif consumer == "repeat_after_sec":
            got = s.repeat_after_sec(T, 0, n)
            kind = prod["flags"] & 7
            want = np.zeros(n, dtype=np.int64)
            iv = (kind == am.KIND_INTERVAL) | (kind == am.KIND_CRON_EVERY)
            want[iv] = prod["ras"][iv]
            for i in np.flatnonzero(kind == am.KIND_CRON_SPEC):
                c = orc.OrcCron(int(prod["minute"][i]), int(prod["hour"][i]), int(prod["dom"][i]),
                                int(prod["month"][i]), int(prod["dow"][i]), 0, 1, int(prod["flags"][i] >> 24))
                want[i] = orc.load().orc_cron_repeat_after_sec(C.byref(c), T)
            np.testing.assert_array_equal(got, want)
        elif consumer == "read":
            dev = s.read(slots)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], orac[name][slots], err_msg=f"read: {name}")
            dev = s.read_range(0, n)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], orac[name], err_msg=f"read_range: {name}")
        T_next = T + 1 if ticked else T
        _assert_tick_equal(am, s.tick(T_next), orc.sweep(orac, T_next), s, orac, n, f"tick after {consumer}")


def test_tick_device_resident_outputs(am, orc, gen):
    import torch
    n = 100_000
    prod, orac = _gen_pair(gen, am, orc, 2, 21, n, T0)
    dev = torch.device("cuda:0")
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        d_idx = torch.empty(n, dtype=torch.int32, device=dev)
        d_act = torch.empty(n, dtype=torch.uint8, device=dev)
        d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        d_st = torch.zeros(16, dtype=torch.int64, device=dev)
        stream = torch.cuda.current_stream()
        s.tick_device(T0, 0, d_idx.data_ptr(), d_act.data_ptr(), n, d_cnt.data_ptr(),
                      d_st.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        wi, wa, ws = orc.sweep(orac, T0)
        cnt = int(d_cnt.item())
        assert cnt == len(wi)
        np.testing.assert_array_equal(d_idx[:cnt].cpu().numpy().astype(np.uint64), wi)
        np.testing.assert_array_equal(d_act[:cnt].cpu().numpy().astype(np.uint32), wa)
        got_stats = dict(zip(am.abi.STAT_FIELDS, [int(v) & ((1 << 64) - 1) for v in d_st.cpu().tolist()]))
        assert got_stats == ws


@pytest.mark.parametrize("config,seed", [(2, 2), (3, 3)])
def test_full_size_10m_equals_the_oracle(am, orc, gen, config, seed):
    """BASELINE configs[1] and configs[2] at FULL size (10 M HealthChecks): the emitted list,
    the action bytes, the statistics and all sixteen columns equal the threaded oracle sweep —
    at T0 (cron + interval arms; config 3: 50 % pending Failed / 25 % Succeeded through the
    remedy gate) and one minute later (nothing pending: the sparse paths)."""
    import os
    n = 10_000_000
    threads = min(32, len(os.sched_getaffinity(0)))
    prod = gen.fill(config, seed, 0, n, T0, am.load().am_healthcheck_classify, threads=threads)
    orac = gen.fill(config, seed, 0, n, T0, orc.load().orc_classify, threads=threads)
    for name in am.COLUMN_NAMES:
        assert np.array_equal(prod[name], orac[name]), f"classify column {name}"
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        for T in (T0, T0 + 60):
            gi, ga, gs = s.tick(T)
            wi, wa, ws = orc.sweep(orac, T, threads=threads)
            assert gs == ws, f"config {config} T={T}: stats differ\n gpu={gs}\n cpu={ws}"
            assert np.array_equal(gi, wi), f"config {config} T={T}: emitted indices"
            assert np.array_equal(ga, wa), f"config {config} T={T}: action bytes"
            # size-independent properties of the list itself
            assert (np.diff(gi.astype(np.int64)) > 0).all()
            assert int(np.bitwise_xor.reduce(gi)) == gs["idx_xor"] and int(gi.sum(dtype=np.uint64)) == gs["idx_sum"]
        dev = s.read_range(0, n)
        for name in am.COLUMN_NAMES:
            assert np.array_equal(dev[name], orac[name]), f"config {config}: column {name} after two ticks"


def test_shard_additivity_at_10m(am, gen):
    """4 index-range shards of the 10 M population concatenated == the whole (SURVEY 8e), and
    re-ticking the same second is idempotent up to the one-shot "Stopped" report."""
    n = 10_000_000
    prod = gen.fill(2, 2, 0, n, T0, am.load().am_healthcheck_classify, threads=8)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        idx, act, st = s.tick(T0)
        idx2, act2, st2 = s.tick(T0)
        keep = (act & ~np.uint32(am.ACT_STOPPED)) != 0
        np.testing.assert_array_equal(idx2, idx[keep])
        assert st2["n_stopped"] == 0 and st["n_stopped"] > 0
    parts = []
    q = n // 4
    for r in range(4):
        cols = {k: np.ascontiguousarray(v[r * q:(r + 1) * q]) for k, v in prod.items()}
        with am.Sweep(capacity=q, shard_base=r * q) as s:
            s.load_range(0, cols)
            parts.append(s.tick(T0)[0])
    np.testing.assert_array_equal(np.concatenate(parts), idx)


def test_timer_armed_conjunct_of_the_ladder(am, orc):
    """hcc.go:264 skips only when "elapsed < RepeatAfterSec && timer != nil".  After a controller
    restart (empty RepeatTimersByName, hcc.go:161) a check that finished one second ago is
    submitted anyway; once its result is applied the timer is armed (hcc.go:745-752) and the
    interval rule holds again."""
    T = T0
    recs, orecs = [], []
    for armed in (True, False):
        for kw in (dict(repeat_after_sec=3600), dict(cron="@every 1h")):
            rc, r = am.classify(finished_at=T - 1, timer_armed=armed, **kw)
            assert rc == 0
            recs.append(r)
    recs = np.concatenate(recs)
    assert [bool(f & am.F_TIMER_ARMED) for f in recs["flags"]] == [True, True, False, False]
    cols = am.records_to_columns(recs)
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=4) as s:
        s.load_range(0, cols)
        got = s.tick(T)
        want = orc.sweep(ocols, T)
        assert got[2] == want[2]
        assert got[0].tolist() == want[0].tolist() == [2, 3]            # only the unarmed pair is due
        assert got[1].tolist() == [am.ACT_SUBMIT_HC] * 2
        s.post_result([2, 3], [am.PHASE_SUCCEEDED, am.PHASE_FAILED])   # results arm the timers ...
        ocols["flags"][2] |= am.F_PENDING_OK
        ocols["flags"][3] |= am.F_PENDING_FAIL
        got = s.tick(T + 1)
        want = orc.sweep(ocols, T + 1)
        assert got[2] == want[2] and len(got[0]) == len(want[0]) == 0   # ... and nothing is due one second later
        dev = s.read_range(0, 4)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], ocols[name], err_msg=name)
        assert all(f & am.F_TIMER_ARMED for f in dev["flags"])


def test_workflow_phase_and_remedy_phase_posted_by_separate_calls(am, orc):
    """The reference observes the two phases in separate watch loops (hcc.go:607-756, :788-852):
    a "Failed" and a remedy "Succeeded" posted by two calls before ONE tick must both take
    effect — and equal the single call carrying both."""
    T = T0
    rc, r = am.classify(repeat_after_sec=3600, finished_at=T - 10, has_remedy=True, remedy_runs_limit=2,
                        remedy_reset_interval=300)
    assert rc == 0
    recs = np.concatenate([r, r, r, r])
    cols = am.records_to_columns(recs)
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=4) as s:
        s.load_range(0, cols)
        s.post_result([0], [am.PHASE_FAILED])                               # slot 0: two calls
        s.post_result([0], [am.PHASE_NONE], [am.PHASE_SUCCEEDED])
        s.post_result([1], [am.PHASE_FAILED], [am.PHASE_SUCCEEDED])         # slot 1: one call
        s.post_result([2], [am.PHASE_NONE], [am.PHASE_FAILED])              # slot 2: remedy first,
        s.post_result([2], [am.PHASE_FAILED])                               #         then the failure
        s.post_result([3], [am.PHASE_SUCCEEDED])                            # slot 3: the later phase wins,
        s.post_result([3], [am.PHASE_FAILED])                               #         a later "none" does not erase
        s.post_result([3], [am.PHASE_NONE])
        for i, bits in ((0, am.F_PENDING_FAIL | am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK),
                        (1, am.F_PENDING_FAIL | am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK),
                        (2, am.F_PENDING_FAIL | am.F_REMEDY_PENDING), (3, am.F_PENDING_FAIL)):
            ocols["flags"][i] |= bits
        got = s.tick(T)
        want = orc.sweep(ocols, T)
        assert got[2] == want[2]
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
        assert got[2]["n_result_fail"] == 4 and got[2]["n_remedy_ok"] == 2 and got[2]["n_remedy_fail"] == 1
        dev = s.read_range(0, 4)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], ocols[name], err_msg=name)
        assert dev["remedy_success"].tolist() == [1, 1, 0, 0] and dev["failed"].tolist() == [1, 1, 1, 1]


def test_next_due_is_the_first_second_at_which_a_tick_emits(am, orc):
    """am_sweep_next_due (SURVEY 8f-1: on-device Next() consumed as a wake-up time): no tick before
    it emits anything, the tick at it does — checked by brute force against the oracle's ticks."""
    T = T0 + 17
    specs = [dict(repeat_after_sec=300), dict(repeat_after_sec=3600), dict(cron="@every 10m"),
             dict(cron="*/7 * * * *"), dict(cron="30 10 * * *"), dict(cron="0 0 1 1 *"), dict(repeat_after_sec=86400)]
    for pick, fin_age in (([0, 1, 2, 4], 5), ([1, 5, 6], 100), ([3, 4, 5], 1), ([5], 1), ([1, 6], 3599)):
        recs = []
        for k in pick:
            rc, r = am.classify(finished_at=T - fin_age, **specs[k])
            assert rc == 0
            recs.append(r)
        cols = am.records_to_columns(np.concatenate(recs))
        with am.Sweep(capacity=len(pick)) as s:
            s.load_range(0, cols)
            nd = s.next_due(T)
            o = {k: v.copy() for k, v in cols.items()}
            want = None
            for t in range(T + 1, T + 4 * 3600):
                if len(orc.sweep({k: v.copy() for k, v in o.items()}, t)[0]):
                    want = t
                    break
            if want is None:  # beyond the brute-force horizon: at least nothing may be due inside it
                assert nd is None or nd >= T + 4 * 3600, (pick, nd)
                continue
            assert nd == want, (pick, fin_age, nd, want)
            if nd - 1 > T:
                assert len(s.tick(nd - 1)[0]) == 0
            assert len(s.tick(nd)[0]) >= 1
    # results posted but not yet applied, an unreported "Stopped" and parse errors are due at once
    for kw in (dict(repeat_after_sec=0), dict(cron="NOT_A_VALID_CRON")):
        rc, r = am.classify(finished_at=T - 1, **kw)
        with am.Sweep(capacity=1) as s:
            s.load_range(0, am.records_to_columns(r))
            assert s.next_due(T) == T + 1
    rc, r = am.classify(finished_at=T - 1, repeat_after_sec=3600)
    with am.Sweep(capacity=4) as s:
        s.load_range(0, am.records_to_columns(r))
        assert s.next_due(T) == T - 1 + 3600
        s.post_result([0], [am.PHASE_FAILED])
        assert s.next_due(T) == T + 1
    with am.Sweep(capacity=4) as s:
        assert s.next_due(T) is None


def test_tick_view_and_last_list(am, orc, gen):
    """am_sweep_tick_view hands out the library's pinned buffer (u32 local indices, u8 actions);
    am_sweep_last_list re-reads the same list in pieces after a short-buffer tick (nothing is lost)."""
    n, base = 50_003, 7_000_000
    prod, orac = _gen_pair(gen, am, orc, 3, 9, n, T0, first=base)
    with am.Sweep(capacity=n, shard_base=base) as s:
        s.load_range(0, prod)
        vi, va, st = s.tick_view(T0)
        wi, wa, ws = orc.sweep(orac, T0, shard_base=base)
        assert st == ws and vi.dtype == np.uint32 and va.dtype == np.uint8
        np.testing.assert_array_equal(vi.astype(np.uint64) + np.uint64(base), wi)
        np.testing.assert_array_equal(va.astype(np.uint32), wa)
        # a short-buffer tick consumes the one-shot actions on the device; the list is still there
        with pytest.raises(am.AmError) as e:
            s.tick(T0 + 60, cap=100)
        assert e.value.code == am.AM_E_NOSPACE
        wi, wa, ws = orc.sweep(orac, T0 + 60, shard_base=base)
        assert e.value.needed == len(wi) > 100
        got_i, got_a, off = [], [], 0
        while True:
            i, a, left = s.last_list(off, 7001)
            got_i.append(i); got_a.append(a)
            off += len(i)
            if left <= 7001:
                break
        np.testing.assert_array_equal(np.concatenate(got_i), wi)
        np.testing.assert_array_equal(np.concatenate(got_a), wa)


def test_staged_events_take_effect_in_call_order(am):
    """Reconcile workers and watch loops call in between two ticks; per slot the
    calls must take effect in order (resolved on the device, csrc/sweep_kernels.cuh)."""
    T = T0
    def rec(ras, fin):
        rc, r = am.classify(repeat_after_sec=ras, finished_at=fin)
        assert rc == 0
        return r
    A, B = rec(60, T - 1000), rec(7, T - 1)          # A is due at T, B is not
    with am.Sweep(capacity=64) as s:
        s.upsert([0], A); s.remove([0])              # created then deleted      -> gone
        s.remove([1]); s.upsert([1], A)              # deleted then re-created   -> present, due
        s.upsert([2], A); s.upsert([2], B)           # two reconciles            -> the later spec
        s.upsert([3], B); s.upsert([3], A)
        s.upsert([4], A)
        s.post_result([4], [am.PHASE_FAILED]); s.upsert([4], B)   # result of the replaced CR is dropped
        s.upsert([5], B); s.post_result([5], [am.PHASE_SUCCEEDED])  # result after the upsert applies
        s.upsert([6], B)
        s.post_result([6], [am.PHASE_SUCCEEDED]); s.post_result([6], [am.PHASE_FAILED])  # last result wins
        s.upsert(np.array([7, 7, 7]), np.concatenate([A, B, A]))  # duplicates inside one call: last wins
        idx, act, st = s.tick(T)
        got = dict(zip(idx.tolist(), act.tolist()))
        assert got == {1: am.ACT_SUBMIT_HC, 3: am.ACT_SUBMIT_HC, 7: am.ACT_SUBMIT_HC}, got
        cols = s.read_range(0, 8)
        assert cols["flags"][0] == am.F_TOMBSTONE
        assert cols["ras"].tolist()[1:8] == [60, 7, 60, 7, 7, 7, 60]
        assert cols["failed"][4] == 0 and cols["finished_at"][4] == T - 1     # dropped result
        assert cols["success"][5] == 1 and cols["finished_at"][5] == T        # applied result
        assert cols["failed"][6] == 1 and cols["success"][6] == 0             # FAILED posted last
        assert st["n_result_ok"] == 1 and st["n_result_fail"] == 1 and s.size == 8
        # marks are cleared: the next tick sees no stale ordering state
        s.post_result([5], [am.PHASE_FAILED])
        _, _, st2 = s.tick(T + 1)
        assert st2["n_result_fail"] == 1 and s.read([5])["failed"][0] == 1


def test_repeat_after_sec_on_device_equals_oracle(am, orc, gen):
    """SURVEY 8f-1: hcc.go:262's RepeatAfterSec = Next(now) - now, evaluated for
    every record on the device, against the oracle's Go-shaped Next()."""
    import ctypes as C
    n = 60_000
    prod, _ = _gen_pair(gen, am, orc, 2, 2, n, T0)
    lib = orc.load()
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        for T in (T0, T0 + 17, T_OCT1 - 1, 1709164799, 4102444799):
            got = s.repeat_after_sec(T, 0, n)
            kind = prod["flags"] & 7
            want = np.zeros(n, dtype=np.int64)
            iv = (kind == am.KIND_INTERVAL) | (kind == am.KIND_CRON_EVERY)
            want[iv] = prod["ras"][iv]
            for i in np.flatnonzero(kind == am.KIND_CRON_SPEC):
                c = orc.OrcCron(int(prod["minute"][i]), int(prod["hour"][i]), int(prod["dom"][i]),
                                int(prod["month"][i]), int(prod["dow"][i]), 0, 1, int(prod["flags"][i] >> 24))
                want[i] = lib.orc_cron_repeat_after_sec(C.byref(c), T)
            np.testing.assert_array_equal(got, want, err_msg=f"T={T}")
            assert (got[kind == am.KIND_CRON_SPEC] != 0).all()
        # a sub-range, and the unsatisfiable schedule (Feb 30): Go's saturated value
        rc, r = am.classify(cron="0 0 30 2 *")
        s.upsert([5], r)
        assert s.repeat_after_sec(T0, 5, 1)[0] == -9223372035


def test_snapshot_restore_resumes_bit_exactly(am, orc, gen):
    """Checkpoint/resume (SURVEY section 5: the CR status in etcd is the reference's checkpoint;
    here: am_sweep_read of every column -> am_sweep_load_range into a fresh handle).  A day
    fragment run in two halves with a destroy/create in between equals the uninterrupted run."""
    n, seed = 40_000, 5
    prod, orac = _gen_pair(gen, am, orc, 55, seed, n, T0)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, prod)
        s.set_seed(seed)
        for k in range(70):
            s.tick(T0 - 10 + k, mode=am.SWEEP_CLOSED_LOOP)
        snap = s.read_range(0, n)                      # checkpoint
    with am.Sweep(capacity=n) as s2:                   # "restart"
        s2.load_range(0, snap)
        s2.set_seed(seed)
        tail = [s2.tick(T0 + 60 + k, mode=am.SWEEP_CLOSED_LOOP) for k in range(70)]
        final = s2.read_range(0, n)
    for k in range(140):
        want = orc.sweep(orac, T0 - 10 + k, mode=1, seed=seed)
        if k >= 70:
            gi, ga, gs = tail[k - 70]
            assert gs == want[2], f"tick {k}"
            np.testing.assert_array_equal(gi, want[0])
            np.testing.assert_array_equal(ga, want[1])
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(final[name], orac[name], err_msg=name)
