/*
 * amsweep.h — C-ABI of libamsweep: the GPU-native (H100) per-tick HealthCheck
 * schedule-evaluation sweep for keikoproj/active-monitor.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  Every entry point
 * names the reference decision it replaces; `hcc.go` abbreviates
 * internal/controllers/healthcheck_controller.go of the reference.
 *
 * Conventions (cgo-friendly):
 *   - plain C, fixed-width integers, flat arrays; no callbacks, no torch types;
 *   - every input is COPIED during the call, the library never retains caller
 *     memory; outputs go to caller-provided buffers (capacity passed in);
 *   - return value: 0 on success, negative AM_E_* on failure; never aborts,
 *     never throws across the boundary;
 *   - per-record anomalies are DATA (action bit AM_ACT_ANOMALY), not failures;
 *   - there is NO CPU fallback: without a CUDA device am_sweep_create fails
 *     with AM_E_DEVICE;
 *   - every am_sweep_* / am_gather_* call makes the handle's device the
 *     calling thread's current CUDA device (cudaSetDevice) and leaves it so.
 */
#ifndef AMSWEEP_H_
#define AMSWEEP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AMSWEEP_ABI_VERSION 2

/* ---- error codes ------------------------------------------------------- */
#define AM_OK 0
#define AM_E_INVAL (-1)       /* NULL pointer, bad argument                   */
#define AM_E_RANGE (-2)       /* value outside the HBM column's domain (N1)   */
#define AM_E_NOSPACE (-3)     /* caller buffer too small; needed size returned */
#define AM_E_DEVICE (-4)      /* CUDA failure; see am_last_error_detail       */
#define AM_E_NOMEM (-5)       /* host or device allocation failed             */
#define AM_E_PARSE (-6)       /* cron spec rejected (robfig error text in err) */
#define AM_E_UNSUPPORTED (-7) /* valid spec the device path does not evaluate
                                 (a 256th distinct CRON_TZ zone): keep it on
                                 the Go path                                  */
#define AM_E_BUSY (-8)        /* second concurrent am_sweep_tick on a handle  */

/* ---- cron (replaces cron.ParseStandard, hcc.go:253; robfig/cron v3.0.1) - */
#define AM_CRON_ERROR 0
#define AM_CRON_SPEC 1  /* SpecSchedule: five uint64 masks, bit 63 = starBit  */
#define AM_CRON_EVERY 2 /* ConstantDelaySchedule: delay_sec > 0               */

#define AM_STAR_BIT (1ull << 63)

typedef struct am_cron {
  uint64_t minute, hour, dom, month, dow; /* robfig SpecSchedule fields      */
  int64_t delay_sec;                      /* ConstantDelaySchedule.Delay / s  */
  int32_t kind;                           /* AM_CRON_*                        */
  int32_t tz_id;                          /* SpecSchedule.Location: 0 = time.Local ==
                                             UTC (distroless image, Dockerfile:25),
                                             else an am_tz_lookup id           */
} am_cron_t;

/* Parse `spec[0..len)` exactly as cron.ParseStandard does.  On a rejected
 * spec returns AM_E_PARSE, sets out->kind = AM_CRON_ERROR and writes the
 * robfig-style message (NUL-terminated, truncated to errcap) into err. */
int am_cron_parse(const char* spec, size_t len, am_cron_t* out, char* err, size_t errcap);

/* Named time zones.  robfig resolves a "TZ=" / "CRON_TZ=" prefix with time.LoadLocation and
 * evaluates the schedule in that zone (parser.go; call site hcc.go:253).  Here a zone is registered
 * once per process under a small id (1..255; "", "UTC" and "Local" are 0: the shipped image runs in
 * UTC) read from the system's TZif files ($ZONEINFO, /usr/share/zoneinfo, ...: Go's search path);
 * am_cron_parse does this by itself and returns the id in am_cron_t.tz_id; classify carries it in
 * the record's flags (AM_F_TZ_SHIFT); each tick evaluates such records against their zone's wall
 * clock on the device.  AM_E_PARSE: unknown zone (robfig: "provided bad location");
 * AM_E_UNSUPPORTED: more than 255 distinct zones in one process. */
int am_tz_lookup(const char* name, size_t len, int32_t* tz_id);
/* UTC offset, seconds east, of a registered zone at a UTC instant (0 for id 0). */
int am_tz_offset(int32_t tz_id, int64_t unix_sec, int32_t* utoff_out);

/* matches(T) of SURVEY Appendix A.7 for one schedule and one UTC second:
 * 1 if a SpecSchedule fires exactly at unix_sec, else 0 (host helper; the
 * device evaluates the same predicate inside the sweep kernel). */
int am_cron_matches(const am_cron_t* c, int64_t unix_sec);

/* Schedule.Next(t) for whole-second t (hcc.go:262): first activation strictly
 * after unix_sec, or INT64_MIN when none within five years (robfig returns the
 * zero time).  UTC only. */
int64_t am_cron_next(const am_cron_t* c, int64_t unix_sec);

/* RepeatAfterSec as hcc.go:262 derives it for a clock reading with a non-zero
 * nanosecond part (SURVEY B.4 N2): whole seconds from floor(now) to Next(now).
 * When Next() finds nothing (Go zero time) Sub saturates and the Go value is
 * int(minDuration/Second)+1 = -9223372035, returned as is. */
int64_t am_cron_repeat_after_sec(const am_cron_t* c, int64_t unix_sec);

/* ---- record schema (SURVEY Appendix B.1) -------------------------------- */
/* flags word */
#define AM_KIND_MASK 0x7u
#define AM_KIND_NO_RESOURCE 0u   /* Workflow.Resource == nil, hcc.go:227       */
#define AM_KIND_STOPPED 1u       /* ras<=0 && cron=="", hcc.go:238             */
#define AM_KIND_INTERVAL 2u      /* ras>0 (cron ignored), hcc.go:264           */
#define AM_KIND_CRON_SPEC 3u     /* ras<=0 && 5-field/descriptor, hcc.go:251   */
#define AM_KIND_CRON_EVERY 4u    /* ras<=0 && "@every d", hcc.go:251           */
#define AM_KIND_PARSE_ERROR 5u   /* ParseStandard error, hcc.go:254-257        */
#define AM_KIND_HOST_FALLBACK 6u /* AM_E_UNSUPPORTED specs (a 256th distinct time
                                    zone): not evaluated on the device          */
#define AM_F_HAS_REMEDY (1u << 3)        /* !RemedyWorkflow.IsEmpty()          */
#define AM_F_PENDING_OK (1u << 4)        /* workflow phase Succeeded posted    */
#define AM_F_PENDING_FAIL (1u << 5)      /* workflow phase Failed posted       */
#define AM_F_REMEDY_PENDING (1u << 6)    /* a remedy outcome is attached       */
#define AM_F_REMEDY_OUTCOME_OK (1u << 7) /* ... and it is Succeeded            */
#define AM_F_TOMBSTONE (1u << 8)         /* removed / never upserted           */
#define AM_F_STOPPED_REPORTED (1u << 9)  /* "Stopped" status already written   */
#define AM_F_TIMER_ARMED (1u << 10)      /* RepeatTimersByName holds a timer for the
                                            check (hcc.go:264 "&& timer != nil";
                                            armed by hcc.go:745-752 after a result) */
#define AM_F_CARRY_SHIFT 11              /* bits 11..15: library-internal.  Action bits of a posted result the
                                          * library applied while draining the staged calls of a tick (before
                                          * that tick's sweep, which emits and clears them): never set in a
                                          * record a caller sees or supplies                                */
#define AM_F_CARRY_MASK (0x1Fu << AM_F_CARRY_SHIFT)
#define AM_F_TZ_SHIFT 24                 /* bits 24..31: time zone of a 5-field schedule
                                            ("CRON_TZ=Zone ..."), 0 = UTC; am_tz_lookup   */
#define AM_F_TZ_MASK (0xFFu << AM_F_TZ_SHIFT)
#define AM_F_FAILP_SHIFT 16              /* closed-loop harness: P(fail)*256   */
#define AM_F_FAILP_MASK (0xFFu << AM_F_FAILP_SHIFT)
/* the flags bits that are the CR's spec: what am_sweep_update_spec takes from its records */
#define AM_F_SPEC_MASK (AM_KIND_MASK | AM_F_HAS_REMEDY | AM_F_FAILP_MASK | AM_F_TZ_MASK)

/* action byte emitted per record per tick (0 = nothing to do) */
#define AM_ACT_SUBMIT_HC 0x01u         /* hcc.go:269-288 submit the workflow   */
#define AM_ACT_RUN_REMEDY 0x02u        /* hcc.go:683/705/714 processRemedy     */
#define AM_ACT_STOPPED 0x04u           /* hcc.go:238-250 write status Stopped  */
#define AM_ACT_PARSE_ERROR 0x08u       /* hcc.go:254-257 warning event+requeue */
#define AM_ACT_REMEDY_SKIP 0x10u       /* hcc.go:692-693                       */
#define AM_ACT_RESET_ON_PASS 0x20u     /* hcc.go:649-660                       */
#define AM_ACT_RESET_ON_INTERVAL 0x40u /* hcc.go:695-704                       */
#define AM_ACT_ANOMALY 0x80u           /* nil RemedyFinishedAt at hcc.go:690   */

/* One HealthCheck as the controller sees it (api/v1alpha1/healthcheck_types.go
 * :32-44 spec, :47-66 status); Go `int` is int64. */
typedef struct am_healthcheck {
  int64_t repeat_after_sec;      /* Spec.RepeatAfterSec                        */
  const char* cron;              /* Spec.Schedule.Cron (not NUL-terminated)    */
  size_t cron_len;               /* 0 == ""                                    */
  int32_t has_resource;          /* Spec.Workflow.Resource != nil              */
  int32_t has_remedy;            /* !Spec.RemedyWorkflow.IsEmpty()             */
  int64_t remedy_runs_limit;     /* Spec.RemedyRunsLimit                       */
  int64_t remedy_reset_interval; /* Spec.RemedyResetInterval                   */
  int64_t finished_at;           /* Status.FinishedAt.Unix()                   */
  int64_t remedy_finished_at;    /* Status.RemedyFinishedAt.Unix()             */
  int32_t finished_at_set;       /* Status.FinishedAt != nil                   */
  int32_t remedy_finished_at_set;
  int64_t success_count, failed_count;
  int64_t remedy_success_count, remedy_failed_count, remedy_total_runs;
  uint32_t fail_p8;              /* closed-loop harness only, 0..255           */
  uint32_t timer_armed;          /* r.GetTimerByName(name) != nil (hcc.go:264):
                                    0 after a controller restart (hcc.go:161 starts
                                    with an empty RepeatTimersByName), so the first
                                    evaluation submits whatever finishedAt says   */
} am_healthcheck_t;

/* One packed record = one element of each SoA column. */
typedef struct am_record {
  uint64_t minute, hour, dom, month, dow;
  int64_t finished_at;        /* nil => 0 (hcc.go:231-235)                     */
  int64_t remedy_finished_at; /* nil => 0 (nil-ness matters: N3)               */
  int32_t ras;                /* RepeatAfterSec | @every delay                 */
  uint32_t flags;
  int32_t runs_limit, reset_interval;
  int32_t success, failed, remedy_success, remedy_failed, remedy_total;
  int32_t wf_timeout;         /* workflow timeout in whole seconds, 0 = none: the effective
                                 timeout of hcc.go:981-985 that the caller sets for
                                 am_sweep_upsert (< 0: AM_E_RANGE).  Only read while the hold
                                 in flight is on (see am_sweep_set_hold_in_flight).  The
                                 classify and ingest calls write 0; am_sweep_read does not
                                 return it; am_sweep_load_range sets it to 0.               */
} am_record_t;

/* Ladder classification at upsert, in the order hcc.go:227 -> 238 -> 251 ->
 * 264 (SURVEY B.2).  Returns AM_OK, AM_E_RANGE (value does not fit the column,
 * N1) or AM_E_UNSUPPORTED (record gets AM_KIND_HOST_FALLBACK).  A cron parse
 * error is NOT a call failure: kind = AM_KIND_PARSE_ERROR, like the reference's
 * per-reconcile error. */
int am_healthcheck_classify(const am_healthcheck_t* hc, am_record_t* out);

/* The same ladder for n HealthChecks at once (SURVEY.md 8f-2, bulk ingest at
 * controller start: the informer's initial list replays every CR through
 * Reconcile, hcc.go:170).  Records are independent, so the batch is split
 * over n_threads host threads (<= 0: one per hardware thread).  rc_out[i]
 * (may be NULL) receives what am_healthcheck_classify returns for record i;
 * the call itself returns AM_OK, or AM_E_INVAL / AM_E_NOMEM.  *n_not_ok (may
 * be NULL) counts records whose rc is not AM_OK. */
int am_healthcheck_classify_batch(const am_healthcheck_t* hcs, uint64_t n, am_record_t* out,
                                  int32_t* rc_out, int n_threads, uint64_t* n_not_ok);

/* HealthCheck manifests as the API server serves them (JSON: one object, an array of objects, or a
 * List with "items") -> packed records, natively: one structural pass, then field extraction by the
 * JSON tags of api/v1alpha1/healthcheck_types.go:32-66 / :88-102 and the ladder, split over n_threads
 * host threads (<= 0: all).  For the informer's initial list at controller start (hcc.go:170) and for
 * restores from a dump.  `timer_armed` is applied to every record (0 after a restart, hcc.go:161).
 * out / rc_out (may be NULL) hold `cap` entries; *n_out = HealthChecks found; AM_E_NOSPACE when
 * cap is too small (nothing written), AM_E_PARSE when the document is not JSON of that shape.
 * rc_out[i]: what am_healthcheck_classify returned, or AM_E_PARSE for a malformed object / time. */
int am_healthcheck_ingest_json(const char* json, size_t len, uint32_t timer_armed, am_record_t* out,
                               int32_t* rc_out, uint64_t cap, uint64_t* n_out, int n_threads);

/* RemedyWorkflow.IsEmpty (api/v1alpha1/healthcheck_types.go:104-106):
 * reflect.DeepEqual against the zero value — note a non-nil empty rbacRules
 * slice is NOT empty. */
int am_remedy_is_empty(size_t generate_name_len, int resource_is_nil, int64_t timeout,
                       int rbac_rules_is_nil);

/* SoA view used by bulk load / upsert / read.  Any pointer may be NULL:
 * on input a NULL column means "all zero", on output "do not read". */
typedef struct am_record_cols {
  uint64_t *minute, *hour, *dom, *month, *dow;
  int32_t* ras;
  uint32_t* flags;
  int64_t* finished_at;
  int32_t *runs_limit, *reset_interval;
  int32_t *success, *failed, *remedy_success, *remedy_failed, *remedy_total;
  int64_t* remedy_finished_at;
} am_record_cols_t;

/* ---- the sweep ---------------------------------------------------------- */
typedef struct am_sweep am_sweep_t;

typedef struct am_tick_stats {
  uint64_t n_records;  /* slots swept (high-water mark of this shard)        */
  uint64_t n_emitted;  /* records with a non-zero action                      */
  uint64_t n_submit_hc, n_run_remedy, n_stopped, n_parse_error;
  uint64_t n_remedy_skip, n_reset_on_pass, n_reset_on_interval, n_anomaly;
  uint64_t n_result_ok, n_result_fail; /* feed metrics.MonitorSuccess/Error,
                                          collector.go:19-31 (workflow=healthCheck) */
  uint64_t n_remedy_ok, n_remedy_fail; /* same vectors, workflow=remedy        */
  uint64_t idx_xor, idx_sum;           /* checksum of emitted global indices   */
} am_tick_stats_t;

#define AM_SWEEP_CLOSED_LOOP 0x1u /* harness: a due record completes instantly
                                     with its preset outcome (SURVEY B.3)     */
#define AM_SWEEP_FULL_SCAN 0x2u   /* read every schedule column even on ticks
                                     where no 5-field cron can fire (sec!=0)  */
#define AM_SWEEP_BLOCKED 0x4u     /* am_sweep_run_ticks only: temporal blocking.  Blocks of consecutive
                                     ticks (96; AMSWEEP_BLOCK_TICKS, at most 128) are evaluated in one pass over the columns,
                                     every record stepped from event to event (its next repeat timer,
                                     hcc.go:751; its next cron minute) — per-tick statistics and the
                                     columns afterwards are identical to tick-by-tick evaluation, but
                                     no per-tick lists are produced                                */
#define AM_SWEEP_CATCH_UP 0x8u    /* catch up on seconds the caller did not tick.  Let P be the second of the
                                     handle's previous tick (every successful am_sweep_tick*, am_gather_tick_view
                                     and am_sweep_run_ticks — its last second — sets it; a tick that returns
                                     AM_E_NOSPACE counts).  A tick at T with this bit evaluates every record as a
                                     plain tick at T does, except that a 5-field schedule is due iff it matches at
                                     SOME second t of (P, T] (a zone-bound one: the zone's wall clock at t, with the
                                     zone's offset at t).  A schedule that fired several times in the window is
                                     emitted once, like a late timer of the reference (hcc.go:751).  Everything
                                     else happens once, at T: interval and "@every" checks, posted results
                                     (finishedAt = T), STOPPED, PARSE_ERROR, the closed-loop completion, the
                                     statistics.  Records are evaluated as they stand after the tick's drain: an
                                     upsert staged during a stall counts from the start of the window.
                                     No previous tick, or T <= P: a plain tick.  T - P > 86400, or a window whose
                                     calendar split exceeds the library's fixed per-zone budget: AM_E_RANGE and
                                     nothing happens (nothing drained, P unchanged) — tick plainly instead.
                                     am_sweep_run_ticks: AM_E_INVAL.                                         */

/* One shard of the record array on one CUDA device.  `capacity` slots are
 * allocated up front; `shard_base` is added to local indices wherever a
 * global index is reported (multi-GPU index-range sharding, SURVEY §8e). */
int am_sweep_create(am_sweep_t** out, int device_id, uint64_t capacity, uint64_t shard_base);
void am_sweep_destroy(am_sweep_t*);

/* Bulk load of a contiguous index range [first, first+n) — informer re-list
 * after (re)start (SURVEY §5 "failure detection / recovery").  The columns are
 * taken as they are: they must be values this library produced
 * (am_healthcheck_classify / am_sweep_read).  In particular
 * AM_F_REMEDY_OUTCOME_OK only has a meaning together with AM_F_REMEDY_PENDING.
 * The time zone of a 5-field schedule (flags bits 24..31) is an id of THIS process's
 * registry (am_tz_lookup, handed out in order of first registration): records read
 * in another process, or before a restart that registered zones in another order,
 * must be re-classified.  A CRON_SPEC record naming an id that is not registered makes
 * this call and am_sweep_upsert return AM_E_INVAL without loading anything.
 * A load is a call in the per-slot order: upserts, removes and post_results staged before it
 * take effect first, so the loaded records replace them (a result posted before the load is
 * dropped, as it is by a later upsert; its workflow phase still releases the slot's hold). */
int am_sweep_load_range(am_sweep_t*, uint64_t first, uint64_t n, const am_record_cols_t* cols);

/* Reconcile of created/updated CRs (hcc.go:170-188): scatter n records to
 * local slots idx[i].  Thread-safe; staged and applied by the next tick. */
int am_sweep_upsert(am_sweep_t*, uint64_t n, const uint64_t* idx, const am_record_t* recs);

/* A spec edit of CRs already placed (hcc.go:170-188 Reconcile after a spec change): the spec of n records
 * (am_healthcheck_classify's am_record_t) for local slots idx[i], WITHOUT the CR's status.  Thread-safe; staged
 * like am_sweep_upsert, in the same per-slot call order, and drained wherever upserts are.
 *   taken from recs[i]: minute..dow, ras, runs_limit, reset_interval, wf_timeout and flags & AM_F_SPEC_MASK;
 *   kept from the slot: finished_at, remedy_finished_at, the five counters, the pending, remedy and timer bits,
 *     the run in flight and its deadline, the wait for admission, the status-change bit and its details;
 *   AM_F_STOPPED_REPORTED stays only while the kind stays AM_KIND_STOPPED (a check the edit pauses is reported once).
 * Per slot, let U be its latest upsert or remove of the drain and S its latest spec update: S after U (or no U)
 * applies on top of U; S before U has no effect.  S on a tombstone (removed, or never upserted or loaded) does
 * nothing and never extends the swept range.  Results posted after U stay valid whatever S does: a spec update
 * never supersedes a result, never ends a hold, and the timeout of a running workflow stays the one it started with.
 * Refusals, with nothing staged: as am_sweep_upsert (AM_E_INVAL, AM_E_RANGE). */
int am_sweep_update_spec(am_sweep_t*, uint64_t n, const uint64_t* idx, const am_record_t* recs);

/* CR deleted (hcc.go:175-186: Stop() its timer): tombstone the slots.  A removed
 * slot reads back as flags == AM_F_TOMBSTONE; its other columns are unspecified
 * until the next upsert.  Staged calls (upsert / remove / post_result) take effect
 * per slot in call order at the next tick, read or load. */
int am_sweep_remove(am_sweep_t*, uint64_t n, const uint64_t* idx);

/* Terminal workflow phases observed by the watch loops (hcc.go:635, :662,
 * :821, :836).  phase / remedy_phase: 0 none, 1 Succeeded, 2 Failed.
 * Thread-safe; staged and applied at the start of the next tick.  Calls from several
 * threads (the reconcile workers, hcc.go:170-188) stage concurrently: a call holds the
 * handle's lock only to reserve its range of the staging arrays, so posting scales with
 * the caller's threads; per slot, calls take effect in the order they entered the library.
 * A call with an out-of-range slot (AM_E_RANGE) or a phase outside 0..2 (AM_E_INVAL) has
 * no effect at all. */
#define AM_PHASE_NONE 0
#define AM_PHASE_SUCCEEDED 1
#define AM_PHASE_FAILED 2
int am_sweep_post_result(am_sweep_t*, uint64_t n, const uint64_t* idx, const uint8_t* phase,
                         const uint8_t* remedy_phase);

/* One tick at wall-clock second unix_sec: drain staged ops, run the sweep
 * kernel, return the ascending list of (global index, action) for every record
 * whose action is non-zero.  Replaces, for every record at once, the decisions
 * at hcc.go:238-267, :649-660, :677-721, :821-851 and the timer at :751.
 * If n_emitted > cap: AM_E_NOSPACE, *n_out = needed, first cap entries valid.
 * Single caller at a time per handle (AM_E_BUSY otherwise). */
int am_sweep_tick(am_sweep_t*, int64_t unix_sec, uint32_t mode, uint64_t* due_idx,
                  uint32_t* due_action, uint64_t cap, uint64_t* n_out, am_tick_stats_t* stats);

/* The same tick without the per-entry pass into caller memory: `view` points at the
 * library's own pinned host buffer, which the GPU wrote directly — u32 LOCAL indices
 * (global = shard_base + idx_local[k]) and u8 actions, ascending.  A cgo caller reads
 * C memory in place (unsafe.Slice).  Valid until the next am_sweep_tick* call on the
 * handle.  Never returns AM_E_NOSPACE. */
typedef struct am_tick_view {
  const uint32_t* idx_local;
  const uint8_t* action;
  uint64_t n;
  uint64_t shard_base;
} am_tick_view_t;
int am_sweep_tick_view(am_sweep_t*, int64_t unix_sec, uint32_t mode, am_tick_view_t* view,
                       am_tick_stats_t* stats);

/* Re-read the list of the last am_sweep_tick / am_sweep_tick_view from entry `offset`
 * on (an AM_E_NOSPACE tick has consumed its one-shot actions — RUN_REMEDY, STOPPED,
 * RESET_* — on the device: fetch the rest here instead of losing them).  *n_out = entries
 * from `offset` to the end; AM_E_NOSPACE again if they exceed cap. */
int am_sweep_last_list(am_sweep_t*, uint64_t offset, uint64_t* due_idx, uint32_t* due_action,
                       uint64_t cap, uint64_t* n_out);

/* Same tick, results left in HBM: launches on `cuda_stream` (a cudaStream_t /
 * CUstream as void*; NULL = CUDA's default stream, as in every CUDA API; use
 * am_sweep_stream() for the handle's own stream) and does not synchronise.
 * d_due_idx (u32 LOCAL indices), d_due_action (u8) hold `cap` entries;
 * d_count receives min(n_emitted, cap) (u32) — the number of valid list entries;
 * d_stats (may be NULL) receives an am_tick_stats_t whose n_emitted is the full count.
 * Alignment: d_due_idx 16 B, d_due_action and d_count 4 B, d_stats 8 B (the kernels store
 * whole quads and words); a misaligned pointer returns AM_E_INVAL before anything happens
 * (nothing drained, the previous tick's second unchanged).  cudaMalloc returns 256-B
 * aligned memory: carve several arrays out of one allocation at such offsets.
 * Used for device-resident pipelines.  Stream rule: every device operation of a handle
 * is ordered after the previous one, whatever streams they were issued on (the library
 * inserts the event waits); a stream passed here must stay alive until the next call on
 * the handle has returned. */
int am_sweep_tick_device(am_sweep_t*, int64_t unix_sec, uint32_t mode, void* d_due_idx,
                         void* d_due_action, uint64_t cap, void* d_count, void* d_stats,
                         void* cuda_stream);

/* Multi-GPU tick, first half: drain + sweep + group scan only.  The emitted set stays
 * inside the handle as a bitmap (1 bit per record) plus the non-default actions;
 * am_gather_exchange ships exactly that over NVLink and rebuilds the GLOBAL list on
 * every GPU.  Two buffer sets alternate, so the exchange of tick k (on another stream)
 * may overlap am_sweep_tick_shard of tick k+1; tick k+2 waits for exchange k by itself.
 * A tick_shard that no exchange follows leaves no statistics behind: a later tick of any
 * entry point counts only its own. */
int am_sweep_tick_shard(am_sweep_t*, int64_t unix_sec, uint32_t mode, void* cuda_stream);

/* Streaming: n_ticks consecutive one-second ticks starting at unix_sec0,
 * back-to-back on the device (BASELINE config 5).  Per-tick stats are written
 * to stats_out[0..n_ticks) (host).  Emitted lists go to an HBM ring and are
 * not copied to the host (with AM_SWEEP_BLOCKED there are none: see above).
 * `seed` keys the closed-loop outcome sequence. */
int am_sweep_run_ticks(am_sweep_t*, int64_t unix_sec0, uint64_t n_ticks, uint32_t mode,
                       uint64_t seed, am_tick_stats_t* stats_out);

/* Simulated workflow durations of am_sweep_simulate, in seconds: 1 <= min <= max for both kinds. */
typedef struct am_sim_params {
  int32_t wf_min, wf_max;          /* health-check workflow duration */
  int32_t remedy_min, remedy_max;  /* remedy workflow duration       */
} am_sim_params_t;

typedef struct am_sim_tick {       /* one row per simulated tick */
  uint64_t n_in_flight;            /* slots am_sweep_in_flight would report after the tick        */
  uint64_t n_remedy_in_flight;     /* slots am_sweep_remedy_in_flight would report after the tick */
  uint64_t n_timed_out;            /* entries am_sweep_last_timed_out would list for the tick     */
  uint64_t n_remedy_timed_out;     /* entries am_sweep_last_remedy_timed_out would list           */
} am_sim_tick_t;

/* A run of n_ticks one-second ticks with the workflows the ticks submit simulated on the device: the
 * hold in flight, the remedy hold and workflow timeouts (INTEGRATION.md §3) over a simulated day.
 * Every draw is a pure function of the run's start second: with g the global index and
 * k = the closed loop's outcome key of (seed, g, start), a health-check run started at S ends Failed iff
 * (k & 0xFF) < the record's fail_p8 (flags bits 16..23), else Succeeded, after
 * wf_min + (k >> 32) % (wf_max - wf_min + 1) seconds; a remedy run started at R ends Succeeded iff
 * ((k >> 8) & 0xFF) < 179 after remedy_min + (k >> 32) % (remedy_max - remedy_min + 1) seconds.
 * For T = unix_sec0 .. unix_sec0 + n_ticks - 1 the call leaves the handle and stats_out[k] exactly as
 *   1. am_sweep_post_result(slot, phase(S), AM_PHASE_NONE) for every slot whose health-check run is held
 *      with start S and S + d(S) <= T, and am_sweep_post_result(slot, AM_PHASE_NONE, rphase(R)) for every
 *      slot whose remedy run is held with start R and R + dr(R) <= T (runs overdue at the first tick
 *      included, whoever started them);
 *   2. am_sweep_tick(h, T, mode & AM_SWEEP_FULL_SCAN, ...), its statistics into stats_out[k] and the
 *      counts above into sim_out[k] (sim_out may be NULL)
 * would, after the calls staged before this one.  So a run whose end equals its deadline completes, and
 * one whose deadline comes first times out and never posts its phase.  Like am_sweep_run_ticks it
 * produces no per-tick lists: afterwards the timed-out lists and the change list are empty, and with
 * tracking on the bits are re-seeded from the flags.  P becomes the last second; runs still in flight
 * stay held for later ticks, am_sweep_in_flight and am_sweep_next_due.  AM_SWEEP_BLOCKED runs the
 * temporal-blocking kernel (blocks as in am_sweep_run_ticks) with the same results.  The seed becomes
 * the handle's (am_sweep_set_seed).  Refused before anything happens (nothing drained, P unchanged):
 * AM_E_INVAL while the hold in flight or the remedy hold is off, for params NULL or out of bounds,
 * stats_out NULL, n_ticks > 2^24 or a mode bit other than AM_SWEEP_BLOCKED | AM_SWEEP_FULL_SCAN;
 * AM_E_RANGE for times out of range. */
int am_sweep_simulate(am_sweep_t*, int64_t unix_sec0, uint64_t n_ticks, uint32_t mode, uint64_t seed,
                      const am_sim_params_t* params, am_tick_stats_t* stats_out, am_sim_tick_t* sim_out);

/* RepeatAfterSec of records [first, first+n) as the reference derives it at
 * reconcile time (hcc.go:259-262): Next(unix_sec) - unix_sec for a 5-field
 * schedule (robfig SpecSchedule.Next evaluated on the device; -9223372035 when
 * nothing fires within five years), the stored interval (whatever its sign) for
 * "@every"/interval checks, 0 otherwise.  On-demand query, not part of the per-tick path. */
int am_sweep_repeat_after_sec(am_sweep_t*, int64_t unix_sec, uint64_t first, uint64_t n, int64_t* out);

/* The earliest second after unix_sec at which a tick of this shard would emit anything or time a
 * run out (workflow timeouts, see am_sweep_set_hold_in_flight: a held run with deadline D counts as
 * an event at max(D, unix_sec + 1), whether or not its expiry emits anything), given
 * the state as it stands (staged events included, no further ones assumed): the wake-up time of
 * the reference's earliest repeat timer (hcc.go:751) or cron activation (hcc.go:262), evaluated on
 * the device over every record (robfig SpecSchedule.Next for 5-field schedules).  The 1 Hz ticker
 * may sleep until then — or until the next upsert / post_result, whichever comes first: ticks in
 * between return an empty list.  INT64_MAX when nothing will ever be due. */
int am_sweep_next_due(am_sweep_t*, int64_t unix_sec, int64_t* next_out);

/* Device -> host read-back of record state (status write-back, hcc.go:1445;
 * checkpoint, SURVEY §5). idx == NULL reads the range [first, first+n). */
int am_sweep_read(am_sweep_t*, uint64_t first, uint64_t n, const uint64_t* idx,
                  am_record_cols_t* out);

/* Hold in flight: one health-check workflow per check at a time, as the reference's watch loop
 * keeps it (hcc.go:607-727 block until the workflow's terminal phase or its timeout; only then
 * hcc.go:745-752 arm the next timer).  Off by default.  While on, the handle keeps per slot
 * `since`, the second of the tick that submitted the check's running workflow, or none.  A record
 * is HELD at a tick when since is set, since >= finishedAt, and no workflow phase (Succeeded /
 * Failed) is pending for it.  A held record gets no AM_ACT_SUBMIT_HC; everything else about it is
 * evaluated as usual (remedy results, RUN_REMEDY and the other one-shot actions, STOPPED,
 * PARSE_ERROR).  Every record a tick emits with AM_ACT_SUBMIT_HC gets since = that tick's second,
 * also in a tick that returns AM_E_NOSPACE (the rest of its list is in am_sweep_last_list).
 * Release: a posted workflow phase clears since when the next tick or read drains it — also when
 * an upsert of the slot staged after it supersedes the result itself, and whatever second the next
 * tick has.  Workflow timeouts (hcc.go:603-632: the watch loop gives up after Spec.Workflow.Timeout
 * and posts a synthetic Failed) are kept on the device, below.  am_sweep_remove and am_sweep_load_range clear since for their slots; a remedy
 * phase alone does not.  An upsert keeps the hold (a status write during a run re-enters
 * Reconcile; it must not submit the check again) unless its finishedAt is later than since.
 * Only the health-check workflow is held unless the remedy hold is on (am_sweep_set_hold_remedy).
 * Works with AM_SWEEP_CATCH_UP, AM_SWEEP_FULL_SCAN, named zones and every tick entry point
 * (am_sweep_tick, _tick_view, _tick_device, _tick_shard and so am_gather_exchange /
 * am_gather_tick_view).  While on, a tick with AM_SWEEP_CLOSED_LOOP and am_sweep_run_ticks return
 * AM_E_INVAL before anything happens (nothing drained, P unchanged).  am_sweep_next_due skips held
 * records: their next event is a post_result or a remove.
 * Turning the hold on starts with nothing in flight (turn it on before the first tick); turning it
 * off makes every slot read as not in flight.  The first call with on != 0 allocates 8 B per slot
 * of capacity on the device.  Replaces the caller's own de-duplication of in-flight checks.
 * Workflow timeouts, while the hold is on: every run a tick submits gets the deadline
 * D = T + W when the slot's wf_timeout W (from its latest upsert) is > 0 at that tick, and none
 * otherwise; a later submission of the slot replaces D, and a remove, a load_range and turning the
 * hold off or on drop it.  So an upsert during a run changes the timeout of the next run only.  The
 * first tick of any entry point with T >= D looks at the run after the tick's drain: if it is still
 * held (a live record), the tick treats it exactly as if am_sweep_post_result(slot,
 * AM_PHASE_FAILED, AM_PHASE_NONE) had been the last call before the tick (FailedCount + 1,
 * finishedAt = T, the timer armed, the remedy gate and its actions, n_result_fail, the hold
 * released, then the due decision at T: a 5-field check that matches T is submitted again in the
 * same tick).  Either way D is dropped: a phase posted before that tick wins, a run released by
 * then is not timed out, and a later upsert that holds it again does not bring D back.  A refused
 * tick times nothing out.  The first upsert with a non-zero wf_timeout allocates 24 B per slot of
 * capacity on the device; handles that never receive one launch nothing more.  Remedy workflows
 * time out only under the remedy hold, and am_sweep_run_ticks is refused while the hold is on
 * anyway.  Turning the hold off also turns the remedy hold off. */
int am_sweep_set_hold_in_flight(am_sweep_t*, int on);

/* Remedy hold: a check is not submitted while its remedy workflow runs, as in the reference, where
 * the Failed branch of the watch loop runs the remedy and blocks in watchRemedyWorkflow until it
 * ends or times out (hcc.go:683-714, :788-852); only then is the status written and the next timer
 * armed.  Without it the check keeps its schedule while the remedy runs, and every failure in that
 * time reads RemedyTotalRuns before the running remedy's phase is posted: a slow remedy can be
 * started many times over its runs limit.  Off by default; AM_E_INVAL (nothing changes) while the
 * hold in flight is off.  While on:
 *  - A remedy run STARTS at a tick T whose action for a check carries AM_ACT_RUN_REMEDY when no
 *    remedy outcome was applied with it (a remedy phase posted in the same call as the Failed, or
 *    in an earlier call before the tick: then the remedy completed at once and nothing is held) —
 *    whether the Failed was posted or is a workflow timeout's, and also in a tick that returns
 *    AM_E_NOSPACE.  Its start is T (RemedyStartedAt, the `then` of hcc.go:790).  With the timeout
 *    state (a non-zero wf_timeout was ever upserted) it gets the deadline D = T + W when the slot's
 *    wf_timeout W is > 0 at T, none otherwise: the remedy watch uses Spec.Workflow.Timeout.
 *  - While it runs the check is HELD: no AM_ACT_SUBMIT_HC, also at the tick T that starts it (a
 *    5-field check matching T at the tick its Failed is applied is not submitted).  Everything
 *    else about it is evaluated as usual.  am_sweep_in_flight reads INT64_MIN for it and
 *    am_sweep_remedy_in_flight its start; am_sweep_next_due skips it and counts D as an event at
 *    max(D, unix_sec + 1).
 *  - It ENDS at the drain of a posted remedy phase (also when a later upsert supersedes the result
 *    itself) or a posted workflow phase (applied as always), at a remove, at am_sweep_load_range
 *    and when either hold is turned off.  An upsert keeps it.  The check is then due by its usual
 *    rule (finishedAt + RepeatAfterSec, or its schedule): one that became due while the remedy ran
 *    is submitted at the tick that ends it.  (The reference re-arms its timer RepeatAfterSec after
 *    the remedy ends, hcc.go:751: a divergence, see INTEGRATION.md section 5.)
 *  - TIMEOUT: the first tick of any entry point with T >= D looks at the run after its drain; if it
 *    is still held on a live record, the tick treats it exactly as if am_sweep_post_result(slot,
 *    AM_PHASE_NONE, AM_PHASE_FAILED) had been the last call before it (RemedyFailedCount + 1,
 *    RemedyTotalRuns = success + failed, RemedyFinishedAt = T, n_remedy_fail, the run ended, then
 *    the due decision at T) and lists it in am_sweep_last_remedy_timed_out.  D is dropped either way.
 * Turning it off ends every remedy run (one pass over the slots); it costs no memory of its own. */
int am_sweep_set_hold_remedy(am_sweep_t*, int on);

/* The remedy runs the last tick timed out (remedy hold): the contract of am_sweep_last_timed_out,
 * with started[k] the run's start (RemedyStartedAt), for the status and the "remedy workflow is
 * timedout" event (hcc.go:813-818) the caller writes. */
int am_sweep_last_remedy_timed_out(am_sweep_t*, uint64_t offset, uint64_t* idx, int64_t* started, uint64_t cap,
                                   uint64_t* n_out);

/* For each slot of [first, first+n) (idx == NULL) or idx[0..n): the start of the slot's running
 * remedy workflow the next tick would hold (remedy hold), INT64_MIN for every other slot (and for all
 * of them while the remedy hold is off).  Drains staged calls like am_sweep_read. */
int am_sweep_remedy_in_flight(am_sweep_t*, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* started_out);

/* Submit budget: the most AM_ACT_SUBMIT_HC entries a tick submits, so that a controller never starts more workflows than
 * it can hand off (DESIGN.md section 6 item 19).  per_tick is the budget of every later tick of every entry point
 * (am_sweep_tick, _tick_view, _tick_device, _tick_shard and so am_gather_exchange / am_gather_tick_view, and each tick
 * of am_sweep_simulate) until it is set again; UINT64_MAX, the default, is unlimited.  AM_E_INVAL, changing nothing,
 * while the hold in flight is off; turning the hold off or on makes it unlimited again and ends every wait below.  The
 * first finite budget allocates about 21.2 B per slot of capacity on the device; a handle that never sets one launches
 * nothing for it.  At a tick T:
 *  - a CANDIDATE is a record the tick would emit with AM_ACT_SUBMIT_HC with an unlimited budget if every record that
 *    waits for admission were due: live, INTERVAL / CRON_EVERY / CRON_SPEC, not held (either hold), and due by its
 *    usual rule (catch-up windows and named zones included) or waiting;
 *  - candidates are admitted in this order: waiting ones by waiting second, then index, then fresh ones by index.  The
 *    first min(budget, candidates) are ADMITTED and get what a submission gets (SUBMIT_HC, since = T, the deadline
 *    T + W), so StartedAt and the workflow timeout count from admission;
 *  - every other candidate is DEFERRED: SUBMIT_HC leaves its entry (an entry left with no action leaves the list; no
 *    other action is budgeted), its since and deadline are none, and it waits from T on unless it already waited.  A
 *    5-field check waiting across several activations is submitted once;
 *  - a wait ends at admission, at a tick at which the record is not a candidate (stopped, parse error, no resource,
 *    removed, held by a remedy run), at a remove, a load, a restore of the slot, a posted workflow phase, and when the
 *    hold is toggled; an upsert keeps it.  A waiting check is admitted after at most ceil(checks ahead / budget) ticks
 *    with a non-zero budget.
 * The tick's list, am_tick_stats_t, n_emitted, the device and shard lists and the exchange are the admitted list's;
 * the result counters are not budgeted.  am_sweep_next_due counts a waiting check as due at unix_sec + 1,
 * am_sweep_in_flight reads INT64_MIN for it, change tracking never lists admission by itself and the details report the
 * action of the admitted list.  The budget is per handle, so per shard.  Refused (AM_E_INVAL, before anything happens):
 * am_sweep_simulate with AM_SWEEP_BLOCKED under a finite budget or while a check waits (as the waits stand after the
 * last drain: calls staged since are not applied by a refused call).  Checkpoints carry the waits (AM_CKPT_ADMISSION)
 * and a restore puts its slots back into the admission order by (waiting second, index); the budget itself is not
 * carried: set it, as the other switches, before restoring. */
int am_sweep_set_submit_budget(am_sweep_t*, uint64_t per_tick);

typedef struct am_admission {
  uint64_t n_candidates;   /* candidates of the last tick                                      */
  uint64_t n_admitted;     /* ... admitted: min(budget, n_candidates)                          */
  uint64_t n_deferred;     /* slots still waiting after it                                     */
  int64_t oldest_deferred; /* the least waiting second among them, INT64_MAX when none waits  */
} am_admission_t;

/* The admission of the last tick of any entry point (after am_sweep_tick_device / am_sweep_tick_shard: waits for it).
 * AM_E_INVAL when the handle never had a finite budget; zero counts after the hold was toggled. */
int am_sweep_last_admission(am_sweep_t*, am_admission_t* out);

/* For each slot of [first, first+n) (idx == NULL) or idx[0..n): the second since which the check waits for admission,
 * INT64_MIN when it does not.  Drains staged calls like am_sweep_in_flight. */
int am_sweep_deferred(am_sweep_t*, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* since_out);

/* The runs the last tick (of any entry point) timed out, ascending by global index, from entry
 * `offset` on: idx[k] the global index, since[k] the run's Status.StartedAt (hcc.go:609/665), for
 * the status and the "Workflow timed out" event (hcc.go:631) the caller writes.  *n_out = entries
 * from `offset` to the end; AM_E_NOSPACE if they exceed cap (the first cap entries are valid);
 * AM_E_RANGE when offset is past the end.  Every tick resets the list (empty while the hold is off
 * or no wf_timeout was ever set); it is valid until the next tick.  After am_sweep_tick_device /
 * am_sweep_tick_shard the call waits for that tick to finish. */
int am_sweep_last_timed_out(am_sweep_t*, uint64_t offset, uint64_t* idx, int64_t* since, uint64_t cap, uint64_t* n_out);

/* For each slot of [first, first+n) (idx == NULL) or idx[0..n): the `since` of a slot the next
 * tick would hold for its health-check run, INT64_MIN for every other slot (and for all of them
 * while the hold is off; a slot whose remedy runs is in am_sweep_remedy_in_flight).
 * Drains staged calls like am_sweep_read.  `since` is the run's Status.StartedAt (`then`,
 * hcc.go:609/638/665), which the caller can write back with the result. */
int am_sweep_in_flight(am_sweep_t*, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* since_out);

/* Sparse state queries: the slots of [first, first+n) in one state, with their value, their count and the least value,
 * found on the device (DESIGN.md section 6 item 22), so that a restart, a stuck-run alert or a gauge need not copy a
 * dense read of every slot to the host.
 *  - A STATE names one dense per-slot query; the value of a slot is what that query returns for it at this point:   */
#define AM_SEL_IN_FLIGHT 1u        /* value = what am_sweep_in_flight returns for the slot        */
#define AM_SEL_REMEDY_IN_FLIGHT 2u /* value = what am_sweep_remedy_in_flight returns for the slot */
#define AM_SEL_WAITING 3u          /* value = what am_sweep_deferred returns for the slot         */
/*  - Slot i of [first, first+n) MATCHES when its value v is not INT64_MIN and v <= before (INT64_MAX: every slot in
 *    the state; T - X: in it since before T - X).
 *  - idx[k] (global index, shard_base added, ascending) and value[k] of the first min(cap, *n_match) matches are
 *    written; *n_match = the matches of the whole range and *oldest = their least value (INT64_MAX when none), also
 *    when the list is cut short.  AM_E_NOSPACE when *n_match > cap (the first cap entries are valid).  With cap == 0,
 *    idx and value may be NULL: the counting form.  Page with a cursor: call again with first = the last returned
 *    local slot + 1 (the call keeps nothing between calls).
 *  - Refused with AM_E_INVAL before the tick guard, nothing drained: an unknown state, n_match or oldest NULL, cap > 0
 *    with idx or value NULL, or a range am_sweep_in_flight refuses.  Otherwise it behaves as am_sweep_in_flight does:
 *    n == 0 returns at once, AM_E_BUSY during a tick, staged calls are drained first, and a tick of
 *    am_sweep_tick_device / am_sweep_tick_shard on a caller stream is waited for.
 *  - While the state is off (the hold, the remedy hold, or the hold with the admission state of a finite budget) the
 *    call returns AM_OK with *n_match = 0 and *oldest = INT64_MAX, and launches nothing beyond its drain.
 *  - Kernel launches of a call that reaches the device: 4 with cap > 0 (the mark pass, the group scan, the
 *    compaction and the gather of min(cap, n) values, whether or not anything matches), 1 with cap == 0.  One
 *    synchronisation.  The first such call allocates about 4.13 B per slot of capacity on the device (a 1-bit mask,
 *    per-group counts and offsets, the list), kept until am_sweep_destroy; a handle that never calls it allocates and
 *    launches nothing for it. */
int am_sweep_select(am_sweep_t*, uint32_t state, uint64_t first, uint64_t n, int64_t before, uint64_t* idx,
                    int64_t* value, uint64_t cap, uint64_t* n_match, int64_t* oldest);

/* Status changes: which checks need their status written back after a tick (the reference writes
 * the status subresource after every phase it applies, updateHealthCheckStatus, hcc.go:734 and
 * :1445-1462).  Off by default.  While on, every tick of every entry point (am_sweep_tick,
 * _tick_view, _tick_device, _tick_shard and so am_gather_exchange / am_gather_tick_view) records
 * its CHANGED SET: the slots whose columns, as am_sweep_read returns them, the tick changed, not
 * counting the library-internal bits AM_F_CARRY_MASK and the posted-result bits AM_F_PENDING_* /
 * AM_F_REMEDY_* the tick consumes.  That is every live record to which the tick applied a
 * workflow result (a posted Succeeded / Failed, a workflow timeout's Failed, a closed-loop
 * completion) or a remedy result (a posted remedy phase, a remedy timeout, an attached outcome),
 * except those whose result the tick reported AM_ACT_ANOMALY (the reference writes no status for
 * them, DESIGN.md section 6 item 5), and every record the tick reported AM_ACT_STOPPED.  Results
 * resolve in the per-slot call order: one superseded by a later upsert or remove is not listed, and
 * one a read's drain left pending belongs to the next tick that applies it.  Upserts, removes,
 * loads, submissions and the holds' bookkeeping are never listed by themselves.  The list is reset
 * by every tick that reaches its drain (a refused tick leaves it; an AM_E_NOSPACE tick records it
 * as usual).  am_sweep_run_ticks does not track its ticks: it empties the list, and the next tick
 * lists only what it changes itself.
 * Turning it on allocates 4.125 B per slot of capacity on the device at the first such call (none
 * for a handle that never turns it on); the first tick after it starts a fresh set.  Turning it off
 * frees nothing; a handle with it off launches nothing for it. */
int am_sweep_set_track_changes(am_sweep_t*, int on);

/* The last tick's changed set (am_sweep_set_track_changes), ascending by global index, from entry
 * `offset` on: idx[k] the global index and, for every non-NULL column of `cols` (cols itself may be
 * NULL), element k the slot's value, gathered on the device (NULL columns are not read, as in
 * am_sweep_read: fetch only what a status write needs).  *n_out = entries from `offset` to the end;
 * AM_E_NOSPACE if they exceed cap (the first cap entries are valid); AM_E_RANGE when offset is past
 * the end; AM_E_INVAL while tracking is off.  After am_sweep_tick_device / am_sweep_tick_shard the
 * call waits for that tick to finish.  It does NOT drain staged calls: the values are the columns
 * as they stand, which are the tick's results unless a call that drains (am_sweep_read,
 * am_sweep_in_flight, am_sweep_next_due, am_sweep_load_range, ...) has applied upserts staged since
 * the tick.  A run's StartedAt is not here: the caller has it from am_work_item_t.unix_sec and the
 * timed-out lists. */
int am_sweep_last_changes(am_sweep_t*, uint64_t offset, uint64_t* idx, am_record_cols_t* cols, uint64_t cap,
                          uint64_t* n_out);

/* Change details: what the last tick applied to each check of its changed set, and the start of
 * the run whose phase it applied, so that a status write and the per-check metrics need no shadow
 * state (hcc.go:627-661, :673-721, :813-851; internal/metrics/collector.go).  One entry per entry
 * of am_sweep_last_changes, same order. */
typedef struct am_change_detail {
  int64_t started;        /* StartedAt of the health-check run whose workflow phase this tick applied, else INT64_MIN */
  int64_t remedy_started; /* RemedyStartedAt of the remedy run whose remedy phase this tick applied, else INT64_MIN */
  uint32_t applied;       /* AM_CHG_* bits */
  uint32_t action;        /* the AM_ACT_* bits the tick emitted for the slot, 0 if it emitted none */
} am_change_detail_t;

#define AM_CHG_SUCCEEDED 0x01u        /* a workflow Succeeded was applied (hcc.go:635-661)             */
#define AM_CHG_FAILED 0x02u           /* a workflow Failed was applied (hcc.go:662-722)                */
#define AM_CHG_TIMED_OUT 0x04u        /* ... that Failed is a workflow timeout's (hcc.go:627-632)      */
#define AM_CHG_REMEDY_SUCCEEDED 0x08u /* a remedy Succeeded was applied (hcc.go:821-835)               */
#define AM_CHG_REMEDY_FAILED 0x10u    /* a remedy Failed was applied (hcc.go:836-851)                  */
#define AM_CHG_REMEDY_TIMED_OUT 0x20u /* ... that remedy Failed is a remedy timeout's (hcc.go:813-818) */
#define AM_CHG_STOPPED 0x40u          /* the tick reported AM_ACT_STOPPED (hcc.go:238-250)            */
#define AM_CHG_CLOSED_LOOP 0x80u      /* the result is the closed-loop harness completion             */

/* Off by default; AM_E_INVAL, changing nothing, while status changes are not tracked (turning
 * tracking off turns details off).  Turning details on applies the calls staged before it, as a
 * read does, and allocates 18 B per slot of capacity on the device at the first such call (none
 * for a handle that never turns them on; a handle with them off launches nothing for them).
 * applied: the posted results the tick applied, as the per-slot call order resolved them (a
 * phase superseded by a later upsert, remove or load is not there; of several phases of one group
 * the latest; a remedy phase merged with the Failed it was posted with or behind; an attached
 * remedy outcome is FAILED | REMEDY_*), plus TIMED_OUT / REMEDY_TIMED_OUT with the Failed of a
 * timeout, STOPPED, and CLOSED_LOOP.  STARTED RULE: with the hold on, started (remedy_started) is
 * what am_sweep_in_flight (am_sweep_remedy_in_flight) would have returned for the slot right
 * before the am_sweep_post_result call that staged the applied workflow (remedy) phase; for a
 * timeout it is the timed-out run's start, for a closed-loop completion T, and otherwise,
 * including whenever the hold is off and for results pending from before details were turned on,
 * INT64_MIN.  action: the slot's entry in the tick's own list. */
int am_sweep_set_change_details(am_sweep_t*, int on);

/* The last tick's change details: out[k] for entry offset + k of am_sweep_last_changes, idx[k]
 * its global index.  Same contract as am_sweep_last_changes (offset, cap, *n_out, AM_E_NOSPACE,
 * AM_E_RANGE; it waits for a device tick and drains nothing); AM_E_INVAL while details are off. */
int am_sweep_last_change_details(am_sweep_t*, uint64_t offset, uint64_t* idx, am_change_detail_t* out, uint64_t cap,
                                 uint64_t* n_out);

/* Checkpoints: a handle's whole state for a range of slots as one self-describing byte blob (DESIGN.md section 6
 * item 19, "Checkpoint format"), so that a restarted or resharded controller goes on tick for tick.  A blob carries,
 * per slot, the sixteen columns (flags bits raw), wf_timeout and the running workflow's deadline when the handle has
 * the timeout state, `since` (remedy runs included) while the hold is on, the change bit while tracking is on and the
 * detail capture while details are on, all as they stand; and the previous tick's second P, the seed, the switches,
 * the names of the time zones its 5-field records use and a 64-bit checksum (against accidental damage, not
 * tampering).  92 B per slot with no switch on, up to 129.125 B with all of them (the waits for admission, 8 B, with
 * AM_CKPT_ADMISSION).  Not carried: the previous tick's
 * lists (am_sweep_last_list, both timed-out lists, the changes and their details: empty on the restored handle until
 * its next tick), profiling state and the launch count.
 * EQUIVALENCE: restore the blobs of one checkpoint of a handle H, all taken between the same two ticks, into handles
 * whose shards cover H's swept slots; from then on the same calls, split by slot, return what they return on H (every
 * tick entry point with its list and statistics except n_records, which is per shard; am_sweep_simulate; read,
 * in_flight, remedy_in_flight, select, repeat_after_sec, next_due; the timed-out lists, the changes and the details).
 * With one handle of the same shard that includes n_records. */
#define AM_CHECKPOINT_VERSION 1
#define AM_CHECKPOINT_VERSION_PACKED 2 /* a packed blob (am_sweep_set_checkpoint_packing) */
#define AM_CKPT_HOLD 0x1u     /* the hold in flight was on                   */
#define AM_CKPT_REMEDY 0x2u   /* ... and the remedy hold                      */
#define AM_CKPT_TRACK 0x4u    /* status changes were tracked                  */
#define AM_CKPT_DETAILS 0x8u  /* ... with change details                      */
#define AM_CKPT_TIMEOUTS 0x10u /* the handle had the workflow-timeout state   */
#define AM_CKPT_ADMISSION 0x20u /* the hold was on and the handle had the submit budget's admission state (a finite
                                   budget was ever set): each slot's waiting second for admission             */
typedef struct am_checkpoint_info {
  uint64_t first_global, n; /* the slots it holds, by GLOBAL index: [first_global, first_global + n)    */
  uint64_t swept_end;       /* global end of the source's swept slots (high-water mark) within the range */
  int64_t prev_tick;        /* P, INT64_MIN when the source had none                                   */
  uint64_t seed;
  uint32_t switches;        /* AM_CKPT_*                                                                */
  uint32_t n_zones;         /* named zones its records use                                              */
  uint32_t version;         /* AM_CHECKPOINT_VERSION                                                    */
  uint32_t reserved;
  uint64_t bytes;           /* the blob's length                                                        */
} am_checkpoint_info_t;

/* Checkpoint of local slots [first, first+n) into buf[0..cap).  A call in the per-slot order: staged calls are drained
 * as am_sweep_read drains them (a result the drain leaves pending is carried pending).  The tick guard is held only
 * while the drain and one device pass over the range are issued on the handle's stream (a tick in that time
 * returns AM_E_BUSY; later ticks queue behind the pass).  The pass packs the sections into a staging area in HBM
 * (allocated at the first checkpoint or restore, about 130 B per slot of capacity, kept until am_sweep_destroy), marks
 * the zones in use and sums the checksum; the copy into buf follows on a stream of its own, while ticks run.
 * Checkpoints and restores of one handle are serialised.
 * *len_out = the blob's length.  AM_E_NOSPACE (after the drain, nothing else done): cap is below what the call needs,
 * returned in *len_out (room for the names of every registered zone; the blob itself may be shorter). */
int am_sweep_checkpoint(am_sweep_t*, uint64_t first, uint64_t n, void* buf, uint64_t cap, uint64_t* len_out);
/* The header of a blob, checked for consistency (format version, sizes, zone table); no handle, no GPU.  The checksum
 * is verified by am_sweep_restore.  AM_E_INVAL: not a blob of this format version, or truncated. */
int am_checkpoint_info(const void* buf, uint64_t len, am_checkpoint_info_t* info);
/* Packed checkpoints (DESIGN.md section 6 item 23, "Packed format"): while `on`, am_sweep_checkpoint,
 * am_sweep_checkpoint_chain and am_sweep_checkpoint_delta write packed blobs (format version 2, the same magics): the
 * version-1 blob's sections cut into blocks of 1024 elements, each encoded on the device in the smallest of five
 * modes (verbatim, one value, frame of reference, sparse, dictionary), with a directory of 16 B per block.  A packed
 * blob is never longer than the version-1 blob plus its directory.  Its header is the version-1 header with version 2,
 * `bytes` its own length, word 14 the version-1 length, and the checksum of the version-1 blob it decodes to, so
 * chains link by content: a raw root may be followed by packed links and the reverse.  While off (the default) they
 * write exactly what they wrote before.  The setting is not handle state: no AM_CKPT_* switch, a restore never needs
 * it, and it may change between the links of a chain.  am_sweep_restore, am_sweep_restore_delta, am_checkpoint_info
 * and am_checkpoint_delta_info take both versions (info.version 1 or 2, info.bytes the blob's own length).
 * A packed blob's length is known only after its encode: a packed checkpoint returns AM_E_NOSPACE (*len_out = the
 * packed length) after its passes, and a refused delta commits nothing.  The encode adds 3 launches to a checkpoint
 * over a non-empty range (sizes, their scan, payloads) on the checkpoint stream after the tick guard is released, and
 * the decode 2 to a restore of a packed blob (directory check, decode).  The packed staging area (about 134 B per slot
 * of capacity) is allocated at the first packed checkpoint or restore and kept until am_sweep_destroy; a handle that
 * never packs allocates and launches nothing for it.  A restore refuses a malformed directory or block (AM_E_INVAL)
 * before anything changes.  Serialised with the handle's checkpoints and restores. */
int am_sweep_set_checkpoint_packing(am_sweep_t*, int on);

/* Restore a blob into this handle: slot g of the blob goes to local slot g - shard_base.  A call in the per-slot order:
 * the calls staged before it are drained first and it replaces them for its slots.  The blob is copied up in chunks,
 * verified on the device (checksum) and its zone names resolved with am_tz_lookup before anything changes; then one
 * pass scatters every section (zone ids rewritten to this process's), the mask planes of the slots are rebuilt, the
 * timeout state is allocated if the blob has it and the handle not (a handle with it restoring a blob without it gets
 * no timeouts and no deadlines for the slots), and the high-water mark is raised to swept_end - shard_base.  P and the
 * seed become the blob's.  Set the switches first, from am_checkpoint_info (am_sweep_set_hold_in_flight, ...).
 * Refused before anything changes (nothing drained, nothing written, P unchanged):
 *   AM_E_INVAL        truncated blob, bad checksum, unknown format version; switches (AM_CKPT_TIMEOUTS aside) that
 *                     differ from the handle's; a handle whose previous tick differs from the blob's P (blobs taken
 *                     at different ticks disagree on P);
 *   AM_E_PARSE        a zone name this process cannot load;
 *   AM_E_UNSUPPORTED  a 256th distinct zone;
 *   AM_E_RANGE        slots outside this shard.
 * Zones registered while resolving the names before a refusal stay registered: the registry is process-wide and only
 * grows, which is harmless. */
int am_sweep_restore(am_sweep_t*, const void* buf, uint64_t len);

/* Delta checkpoints (DESIGN.md section 6 item 21, "Delta format"): a chain over a range of slots is one full blob, its
 * root, then links that carry only the slots whose state changed since the link before.  A standby handle restores the
 * root with am_sweep_restore and applies each delta in order with am_sweep_restore_delta; it then answers as a
 * restore of a full checkpoint taken on the source at the last delta would (EQUIVALENCE above), so a full checkpoint
 * of the range on it is byte for byte the source's.  "Changed" is state-based: a slot is in a delta iff any element a
 * full blob carries for it (the sixteen columns with the flags bits raw, wf_timeout and deadline, since, the change
 * bit, the detail capture, the waiting second) differs from the previous link's, whichever call or tick wrote it.
 * A delta's header holds the chain's range, swept_end, P and the seed at the delta, the switches, n_changed, the
 * link's sequence number (the root is 0), the parent's P and the parent link's checksum; then the n_changed slot
 * offsets (u32, relative to the range's first slot, strictly ascending), every section of the root as an array over
 * those slots only (the change bit packed as bits), and the zone table of their records.  Its magic differs from a
 * full blob's: am_checkpoint_info and am_sweep_restore refuse it (AM_E_INVAL).
 * Memory: a producer reserves, when its first chain starts, a base image of a full blob's sections over its capacity
 * (the previous link's state, up to 129.125 B per slot), the diff's bitmap (1 bit per slot) and the offsets of a
 * delta with every slot changed (4 B per slot); a standby reserves the offsets (4 B per slot) at its first
 * am_sweep_restore_delta.  All are kept until am_sweep_destroy; a handle that never starts a chain or applies a delta
 * allocates nothing and launches nothing for them. */
typedef struct am_checkpoint_delta_info {
  uint64_t first_global, n; /* the chain's range, by GLOBAL index                                     */
  uint64_t swept_end;       /* global end of the source's swept slots within the range, at the delta */
  int64_t prev_tick;        /* P at the delta, INT64_MIN when the source had none                     */
  uint64_t seed;
  uint64_t n_changed;       /* slots it carries                                                       */
  uint64_t seq;             /* the link's sequence number: 1 for the first delta after the root       */
  int64_t parent_prev_tick; /* P of the link before it                                                */
  uint64_t parent_checksum; /* checksum of the link before it (a root's header checksum for seq 1)    */
  uint64_t checksum;        /* its own checksum: the next delta's parent_checksum                     */
  uint32_t switches;        /* AM_CKPT_*, the root's                                                  */
  uint32_t n_zones;
  uint32_t version;         /* AM_CHECKPOINT_VERSION                                                  */
  uint32_t reserved;
  uint64_t bytes;           /* the blob's length                                                      */
} am_checkpoint_delta_info_t;
/* A full checkpoint of local slots [first, first+n) that also starts (or restarts) the handle's delta chain over that
 * range: the blob is byte for byte what am_sweep_checkpoint(first, n) returns at the same point, and its sections stay
 * in HBM as the chain's base.  Same contract and refusals as am_sweep_checkpoint; a refused call leaves the previous
 * chain as it was.  Launches: those of am_sweep_checkpoint (its drain's, and 1 over a non-empty range). */
int am_sweep_checkpoint_chain(am_sweep_t*, uint64_t first, uint64_t n, void* buf, uint64_t cap, uint64_t* len_out);
/* The chain's next link: the slots of its range whose state differs from the previous link's, into buf[0..cap).  A call
 * in the per-slot order that drains as am_sweep_checkpoint does; the tick guard is held only while the drain and the
 * device passes are issued on the handle's stream (the diff against the base image, the compaction and the pack).
 * The copy into buf and the commit of the delta into the base image follow on the checkpoint stream while ticks run;
 * the base advances only once buf holds the blob.  Serialised with checkpoints and restores of the handle.
 * *len_out = the blob's length, *n_changed = the slots it carries.  Launches over a non-empty range: 4 (diff,
 * group scan, compaction, pack) and 1 more (commit) when n_changed > 0, besides its drain's.
 *   AM_E_NOSPACE  (after the drain and the passes) cap is below the blob's length, returned in *len_out; nothing is
 *                 committed: the next delta carries the same slots and whatever changed since;
 *   AM_E_INVAL    the handle has no chain, or its switches (the timeout state included, which a later upsert may
 *                 allocate) differ from the root's: start a new chain. */
int am_sweep_checkpoint_delta(am_sweep_t*, void* buf, uint64_t cap, uint64_t* len_out, uint64_t* n_changed);
/* The header of a delta, checked for consistency (format version, sizes, zone table); no handle, no GPU.  AM_E_INVAL:
 * not a delta of this format version, or truncated. */
int am_checkpoint_delta_info(const void* buf, uint64_t len, am_checkpoint_delta_info_t* info);
/* Apply a delta to this handle.  The handle keeps, per chain range, the checksum of the last link it applied: a full
 * blob restored with am_sweep_restore starts the entry of its range (and drops every entry whose range overlaps it).
 * A delta applies only when an entry exists for its exact range, that entry's checksum is the delta's parent checksum,
 * no tick of any entry point ran on the handle since the entry was last updated, and the handle's P is the delta's
 * parent P or its own P (so several chains taken at the same ticks apply to one handle in any order).  A call in the
 * per-slot order: the calls staged before it are drained first.  Then its slots are scattered (zone ids rewritten to
 * this process's), the mask planes of their segments rebuilt, the high-water mark raised to swept_end - shard_base,
 * the admission order rebuilt when the handle has the admission state, P and the seed set to the delta's and the
 * previous tick's lists emptied, as am_sweep_restore does.  Launches: 4 when n_changed > 0 (offsets and sections
 * verified, scatter, plane rebuild), none otherwise, besides those of its drain, of the allocation of the timeout
 * state when the delta has it and the handle not, and of the admission order's rebuild when the handle has the
 * admission state.  Refused before anything changes, with am_sweep_restore's codes
 * (header, checksum and offsets verified on the device, zone names, switches, slots outside the shard), and:
 *   AM_E_INVAL  offsets that are not strictly ascending below n; no entry for the range, a parent checksum that is
 *               not the entry's (a skipped, repeated or foreign link), a tick since the parent, or a P that is neither
 *               the delta's nor its parent's.  A caller that loses a delta has broken its chain: it starts a new one. */
int am_sweep_restore_delta(am_sweep_t*, const void* buf, uint64_t len);

/* Introspection */
uint64_t am_sweep_size(const am_sweep_t*);     /* high-water mark (slots swept) */
uint64_t am_sweep_capacity(const am_sweep_t*);
int am_sweep_device(const am_sweep_t*);
/* Device time of the last am_sweep_tick / am_sweep_run_ticks sweep kernels
 * (CUDA events on the launching stream), milliseconds; <0 if none. */
double am_sweep_last_kernel_ms(const am_sweep_t*);
/* Per-kernel device timing: when on, every tick records CUDA events on the
 * launching stream before and after sweep_tick_kernel and after the rest of the
 * tick (scan + expand + publish, and before them the submit budget's admission passes
 * when the handle has them).  am_sweep_last_profile waits for the last tick and
 * returns the two durations in milliseconds.  Off by default (the extra events
 * break the programmatic launch chain: do not time a step with it on). */
int am_sweep_set_profiling(am_sweep_t*, int on);
int am_sweep_last_profile(am_sweep_t*, double* sweep_ms, double* rest_ms);
/* Number of kernels this library has launched on the handle so far. */
uint64_t am_sweep_launch_count(const am_sweep_t*);
/* Raw device pointer of a column (for zero-copy wrapping by torch / NCCL
 * plumbing); column ids follow am_record_cols_t member order, 0..15.
 * The five cron-mask columns (0..4) and the kind and zone-id bits of the flags
 * column (AM_KIND_MASK, AM_F_TZ_MASK) must not be written through this
 * pointer: the on-minute sweep reads the masks as bit planes (one bitmap over the
 * shard per value a field can take) that only am_sweep_load_range, upserts and
 * removes keep up to date.  The other flag bits and the other columns may be.
 * Handing out ras (5) or finished_at (7) switches the handle, for good, from the
 * 4-B due word per record the open-loop tick otherwise decides interval checks
 * from back to reading both columns (16 B per record): the library cannot see a
 * write through the pointer, so it stops relying on a word derived from them. */
void* am_sweep_column_ptr(am_sweep_t*, int column);
int am_sweep_set_seed(am_sweep_t*, uint64_t seed);
/* The handle's own non-blocking stream (cudaStream_t as void*). */
void* am_sweep_stream(am_sweep_t*);

/* ---- multi-GPU: the global due list on every GPU, over NVLink peer memory (SURVEY §8e) --
 * One am_gather per rank (one process per GPU).  Every rank creates its exchange block,
 * exports a CUDA-IPC handle, the handles are exchanged by the caller's plumbing
 * (torch.distributed / any side channel) and connected, and the shard layout is set.
 * Then, per tick, every rank calls
 *     am_sweep_tick_shard(sweep, T, mode, stream_a);      // sweep + group scan
 *     am_gather_exchange(gather, sweep, d_stats, stream_b);
 * The exchange ships the sweep's own output — one bit per record for the emitted set,
 * group offsets, the non-default actions — into every peer's block (one kernel, 16-B peer
 * stores, no NCCL, no host round-trip) and rebuilds the GLOBAL ascending (index, action)
 * list locally from the world's bitmaps.  When its last kernel retires, out_idx / out_act
 * on EVERY rank hold that list, out_counts[0..world) the per-rank counts and
 * out_counts[world] the total; d_stats (may be NULL) receives this shard's am_tick_stats_t.
 * stream_b may differ from stream_a (the library orders them): the exchange of tick k then
 * overlaps the sweep of tick k+1.
 * Like any collective, the exchange is a rendezvous: every rank must call it the same
 * number of times.  Its device-side wait for the peers is bounded (AMSWEEP_PUSH_TIMEOUT_MS,
 * default 5000, 0 = unbounded): a peer that never arrives leaves out_counts[world] ==
 * 0xFFFFFFFF and the handle out of step (recreate it).  Argument errors are reported before
 * anything that the peers could observe happens.
 * The reference has no counterpart (single process; consumer is hcc.go:502). */
#define AM_IPC_HANDLE_BYTES 64
typedef struct am_gather am_gather_t;
/* cap_total: records of all shards together (bounds the global list).
 * idx_bytes: 8 = u64 global indices in the output; 4 = u32 (the caller guarantees every
 * global index < 2^32). */
int am_gather_create(am_gather_t** out, int device, int rank, int world, uint64_t cap_total,
                     int idx_bytes);
int am_gather_export(am_gather_t*, void* handle_out /* AM_IPC_HANDLE_BYTES */);
int am_gather_connect(am_gather_t*, const void* handles /* world x AM_IPC_HANDLE_BYTES, rank order */);
/* bases[r] / sizes[r] = first global index / number of records of rank r's shard (the same
 * arrays on every rank).  Required before am_gather_exchange. */
int am_gather_set_layout(am_gather_t*, const uint64_t* bases, const uint64_t* sizes);
int am_gather_exchange(am_gather_t*, am_sweep_t* shard, void* d_stats, void* cuda_stream);
/* One whole step of a sharded controller in one call — the multi-GPU counterpart of am_sweep_tick_view:
 * am_sweep_tick_shard of the bound shard on `sweep_stream` (draining what was posted to it), the
 * exchange on `exchange_stream`, then THIS rank's own part of the global list — its checks, as local
 * slots — extracted into the library's pinned host buffer; one synchronisation.  am_gather_bind names
 * the shard and the two streams once; the view is valid until the next call.  AM_E_DEVICE when a peer
 * did not arrive within AMSWEEP_PUSH_TIMEOUT_MS.  (The global list itself stays on the device:
 * am_gather_out_idx / _act / _counts.) */
int am_gather_bind(am_gather_t*, am_sweep_t* shard, void* sweep_stream, void* exchange_stream);
int am_gather_tick_view(am_gather_t*, int64_t unix_sec, uint32_t mode, am_tick_view_t* view, am_tick_stats_t* stats);
/* Round-1 "plain" format, kept as the measured baseline: every rank writes its FINISHED
 * list (the output of am_sweep_tick_device: u32 local indices, u8 actions, device count)
 * straight into every peer's output buffer at its global offset, 5 or 9 bytes per entry
 * on the wire.  Unbounded device-side waits. */
int am_gather_push(am_gather_t*, const void* d_idx_local /* u32 */, const void* d_act_local /* u8 */,
                   const void* d_count_local /* u32 */, uint64_t shard_base, void* cuda_stream);
void* am_gather_out_idx(am_gather_t*);    /* u64|u32[cap_total], valid after the last exchange / push retires */
void* am_gather_out_act(am_gather_t*);    /* u8[cap_total]                                    */
void* am_gather_out_counts(am_gather_t*); /* u32[world+1]                                     */
/* Device timing of one exchange (CUDA events on its stream): the NVLink push (including the
 * wait for the peers), the list rebuild (counts + expand), the statistics publication. */
int am_gather_set_profiling(am_gather_t*, int on);
int am_gather_last_profile(am_gather_t*, double* push_ms, double* rebuild_ms, double* publish_ms);
const char* am_gather_last_error(const am_gather_t*);
void am_gather_destroy(am_gather_t*);

/* ---- hand-off to the workflow side (SURVEY.md 8f-3; host only, no GPU) ---- */
/* The step AFTER the path: the 1 Hz ticker goroutine publishes the list one
 * am_sweep_tick returned; up to MaxParallel workers (hcc.go:138, the
 * MaxConcurrentReconciles of hcc.go:298) pop chunks and run
 * createSubmitWorkflow / processRemedy (hcc.go:502, :759) for them.  It
 * replaces the goroutine-per-timer fan-out of hcc.go:751 by a bounded FIFO:
 * back-pressure instead of unbounded goroutines when the cluster is slow.
 * Thread-safe for any number of publishers and poppers; never blocks. */
typedef struct am_handoff am_handoff_t;
typedef struct am_work_item {
  uint64_t idx;     /* global record index                                    */
  int64_t unix_sec; /* the tick that emitted it                               */
  uint32_t action;  /* AM_ACT_* bits (already filtered by the publish mask)   */
  uint32_t reserved;
} am_work_item_t;

int am_handoff_create(am_handoff_t** out, uint64_t capacity /* work items */);
void am_handoff_destroy(am_handoff_t*);
/* Enqueue, in order, the entries of one tick whose action has a bit of
 * action_mask set (e.g. AM_ACT_SUBMIT_HC | AM_ACT_RUN_REMEDY).  All or
 * nothing: AM_E_NOSPACE when they do not fit, nothing enqueued, *n_out = the
 * number that would have been; AM_OK: *n_out = number enqueued. */
int am_handoff_publish(am_handoff_t*, int64_t unix_sec, uint64_t n, const uint64_t* idx,
                       const uint32_t* action, uint32_t action_mask, uint64_t* n_out);
/* Dequeue up to `max` items in FIFO order (0 items is not an error). */
int am_handoff_pop(am_handoff_t*, uint64_t max, am_work_item_t* out, uint64_t* n_out);
/* Queue depth and lifetime totals (any pointer may be NULL). */
int am_handoff_stats(am_handoff_t*, uint64_t* pending, uint64_t* published, uint64_t* popped,
                     uint64_t* rejected_batches);

/* UTC broken-down time exactly as the kernel computes it (test hook):
 * out[0..6) = sec, min, hour, dom(1-31), month(1-12), dow(0=Sunday). */
void am_civil_from_unix(int64_t unix_sec, int32_t out[6]);

const char* am_strerror(int code);
const char* am_last_error_detail(const am_sweep_t*); /* NULL handle: create-time error */
int am_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* AMSWEEP_H_ */
