// sweep_kernels.cuh — the per-tick schedule-evaluation sweep for sm_90a (H100).
//
// One launch evaluates every HealthCheck record of a shard at one wall-clock
// second T (SURVEY.md Appendix B.3).  It replaces, for N records at once, the
// per-CR decisions of the reference controller (hcc.go = internal/controllers/
// healthcheck_controller.go):
//     hcc.go:227        Workflow.Resource == nil      -> record skipped
//     hcc.go:238-250    pause rule                    -> AM_ACT_STOPPED
//     hcc.go:251-263    cron arm (robfig bitmasks)    -> matches(T), A.7
//     hcc.go:264, :751  interval / timer              -> T - finishedAt >= ras
//     hcc.go:635-661    Succeeded transition          -> apply_result()
//     hcc.go:662-722    Failed transition + remedy gate
//     hcc.go:821-851    remedy result counters
//
// Shape of the kernel (pure integer work, HBM-bandwidth bound, no tensor cores):
//   * records live as SoA columns in HBM; a CTA of 256 threads owns one tile of
//     1024 consecutive records, a warp owns 128 of them;
//   * every warp-level load instruction is fully coalesced: lane L reads the
//     16 B (two u64 records) or 8 B (two i32 records) at column + (w + 2L),
//     twice per tile ("halves"), plus one 16-B warp-uniform load per cron-mask
//     bit plane, all in flight before the first use (a __syncwarp() after them
//     keeps ptxas from delaying half of them).  Staging the tile in shared memory instead —
//     per-lane cp.async, TMA bulk copies one-shot, and a persistent two-stage
//     TMA pipeline — was built, verified and measured slower for this
//     streaming, near-issue-bound kernel (DESIGN.md section 3);
//   * the tick's broken-down time is computed once per tick as one-hot words
//     and reaches every CTA through the kernel parameters (constant bank); a
//     5-field schedule fires iff minute&M && hour&H && month&Mo && dayMatches
//     (five ANDs, no loop) — on the minute evaluated 32 records per word from
//     the six bit planes (MaskPlanes) those words select;
//   * remedy/counter columns are touched only by lanes whose record has a
//     posted result (or is due, in closed-loop mode): 16 B/record otherwise (8 B in the open-loop
//     variants that read the due words instead of ras and finishedAt, DUE), plus 0.75 B of mask
//     planes on the minute;
//   * the emitted set leaves the kernel as a BITMAP (one bit per record: the four
//     warp ballots the kernel takes anyway, interleaved into four 32-record words
//     per warp, one 128-B line per tile) plus a per-tile list of EXCEPTIONS — the
//     few records whose action is anything but the bare AM_ACT_SUBMIT_HC; no
//     dependency between CTAs.  scan_groups_kernel (one CTA) turns the per-group
//     popcounts into exclusive offsets and expand_kernel rebuilds the contiguous
//     ascending (index, action) list from bitmap + exceptions — for the local shard
//     or, on several GPUs, for every rank's bitmap after the NVLink exchange
//     (gather_kernels.cuh): 1 bit per record crosses the wire instead of 5 bytes per
//     entry.  Round 1 wrote (u32, u8) segments and compacted them (16.7 MB written +
//     33 MB moved per tick at the bench density); a single-pass decoupled look-back was
//     measured before that and rejected;
//   * per-tick statistics are reduced lane -> warp (redux) -> CTA -> global (fire-and-
//     forget RED); kernel boundaries (programmatic dependent launches) are the only
//     global synchronisation, so the sweep kernel has one __syncthreads, no fences and
//     no completion tickets.
#pragma once
#ifndef AMSWEEP_EMULATE  // tests/emu compiles this file for the CPU (cuda_emu.h supplies the model)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/amsweep.h"
#include "civil.h"

#include "sweep_types.h"

namespace amsweep {

// ---- streaming loads / stores: every byte is touched once per tick --------
template <typename T>
__device__ __forceinline__ T ld_stream(const T* p) { return __ldcs(p); }
template <typename T>
__device__ __forceinline__ void st_stream(T* p, T v) { __stcs(p, v); }

// Segment entries are written once by the sweep and read once, a few tens of
// microseconds later, by expand_kernel: keep them L2-resident (evict_last)
// while 560 MB of evict_first column data streams past them.
#ifndef AMSWEEP_EMULATE
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void st_keep_u32(uint32_t* p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_keep_u8(uint8_t* p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u8 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
// programmatic dependent launch (sm_90+): see AM_LAUNCH_PDL
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#else  // CPU emulation: plain stores, the cache policy has no meaning
inline void pdl_wait() {}
inline void pdl_trigger() {}
inline uint64_t l2_evict_last_policy() { return 0; }
inline void st_keep_u32(uint32_t* p, uint32_t v, uint64_t) { *p = v; }
inline void st_keep_u8(uint8_t* p, uint32_t v, uint64_t) { *p = (uint8_t)v; }
#endif

// ---- the posted-result bits of the flags word ---------------------------------
constexpr uint32_t kHcBits = AM_F_PENDING_OK | AM_F_PENDING_FAIL;               // a workflow phase
constexpr uint32_t kRemedyBits = AM_F_REMEDY_PENDING | AM_F_REMEDY_OUTCOME_OK;  // a remedy phase and its outcome
constexpr uint32_t kPendBits = kHcBits | AM_F_REMEDY_PENDING;                   // any posted result

// ---- warp collectives (every lane calls them): the inclusive prefix sum of v over lanes 0 .. lane
__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t up = __shfl_up_sync(kFull, v, d);
    if (lane >= d) v += up;
  }
  return v;
}
// the least v of the warp, in every lane
__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(kFull, v, o);
    v = u < v ? u : v;
  }
  return v;
}
// four 8-bit counters per lane (byte q: counter q) summed over the warp: .x = 0 | 1 << 16, .y = 2 | 3 << 16
__device__ __forceinline__ uint2 warp_byte_sums(uint32_t c) {
  const uint32_t lo = __reduce_add_sync(kFull, (c & 0xFFu) | ((c & 0xFF00u) << 8));
  const uint32_t hi = __reduce_add_sync(kFull, ((c >> 16) & 0xFFu) | ((c >> 8) & 0xFF0000u));
  return make_uint2(lo, hi);
}

__device__ __forceinline__ uint64_t sm64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t outcome_key(uint64_t seed, uint64_t gidx, uint64_t t) {
  return sm64(sm64(seed ^ sm64(gidx)) + t);
}

// the low 16 bits of x -> the even bit positions of a 32-bit word
__device__ __forceinline__ uint32_t spread16(uint32_t x) {
  x &= 0xFFFFu;
  x = (x | (x << 8)) & 0x00FF00FFu;
  x = (x | (x << 4)) & 0x0F0F0F0Fu;
  x = (x | (x << 2)) & 0x33333333u;
  x = (x | (x << 1)) & 0x55555555u;
  return x;
}

// bit i of a 4-bit value -> byte i of a word (0/1 each)
__device__ __forceinline__ uint32_t spread4(uint32_t v) { return ((v & 0xFu) * 0x00204081u) & 0x01010101u; }

// Mutable per-record state carried through the result state machine.
struct RecState {
  uint32_t flags;
  int64_t fa;       // finishedAt
  int32_t s, f;     // SuccessCount, FailedCount
  int32_t rs, rf, rt;  // RemedySuccessCount, RemedyFailedCount, RemedyTotalRuns
  int64_t rfa;      // RemedyFinishedAt, 0 == nil
  int32_t limit, reset;
};

// watchRemedyWorkflow result, hcc.go:821-851
__device__ __forceinline__ void remedy_result(RecState& r, int64_t T, bool ok, uint32_t& res) {
  if (ok) { r.rs = (int32_t)((uint32_t)r.rs + 1u); res += 1u << 16; }
  else    { r.rf = (int32_t)((uint32_t)r.rf + 1u); res += 1u << 24; }
  r.rt = (int32_t)((uint32_t)r.rs + (uint32_t)r.rf);
  r.rfa = T;
}

// Step 1 of B.3: apply a posted workflow result.  Returns action bits; `res`
// counts {ok, fail, remedy_ok, remedy_fail} in its four bytes (a record can
// take two results in one closed-loop tick) for the metrics counters.
__device__ __forceinline__ uint32_t apply_result(RecState& r, int64_t T, uint32_t& res) {
  uint32_t act = 0;
  const uint32_t f = r.flags;
  // watchWorkflowReschedule re-arms the repeat timer after either outcome (hcc.go:745-752)
  const uint32_t armed = (f & kHcBits) ? AM_F_TIMER_ARMED : 0u;
  if (f & AM_F_PENDING_OK) {  // hcc.go:635-661
    r.s = (int32_t)((uint32_t)r.s + 1u);
    r.fa = T;
    res += 1u;
    if ((f & AM_F_HAS_REMEDY) && r.rt >= 1) {  // :649
      r.rt = r.rs = r.rf = 0;
      r.rfa = 0;
      act |= AM_ACT_RESET_ON_PASS;
    }
  } else if (f & AM_F_PENDING_FAIL) {  // hcc.go:662-722
    r.f = (int32_t)((uint32_t)r.f + 1u);
    r.fa = T;
    res += 1u << 8;
    if (f & AM_F_HAS_REMEDY) {  // :677
      bool run = false;
      if (r.limit != 0 && r.reset != 0) {  // :679
        if (r.limit > r.rt) {               // :681
          run = true;
        } else if (r.rfa == 0) {
          act |= AM_ACT_ANOMALY;  // nil RemedyFinishedAt at :690 (N3)
        } else {
          // int(now.Sub(RemedyFinishedAt).Seconds()): Sub saturates at
          // +-9223372036 s, far outside the i32 resetInterval domain
          int64_t d = (int64_t)((uint64_t)T - (uint64_t)r.rfa);
          d = d > 9223372036ll ? 9223372036ll : (d < -9223372036ll ? -9223372036ll : d);
          if ((int64_t)r.reset >= d) {  // :692
            act |= AM_ACT_REMEDY_SKIP;
          } else {  // :695-704
            r.rt = r.rs = r.rf = 0;
            r.rfa = 0;
            act |= AM_ACT_RESET_ON_INTERVAL;
            run = true;
          }
        }
      } else {  // :712-719
        run = true;
      }
      if (run) {
        act |= AM_ACT_RUN_REMEDY;
        if (f & AM_F_REMEDY_PENDING) remedy_result(r, T, (f & AM_F_REMEDY_OUTCOME_OK) != 0, res);
      }
    }
  } else if (f & AM_F_REMEDY_PENDING) {  // remedy finished on its own
    remedy_result(r, T, (f & AM_F_REMEDY_OUTCOME_OK) != 0, res);
  }
  r.flags = (f & ~(kHcBits | kRemedyBits)) | armed;
  return act;
}

// apply_result, and in the closed-loop harness (SURVEY §8d config 5) a record due at T then completes in
// the same tick: the outcome keyed by (seed, global index, T) is posted and applied as well.
template <bool CLOSED>
__device__ __forceinline__ uint32_t result_step(RecState& r, int64_t T, bool due, uint64_t seed, uint64_t g, uint32_t& res) {
  uint32_t act = apply_result(r, T, res);
  if (CLOSED && due) {
    const uint64_t k = outcome_key(seed, g, (uint64_t)T);
    const uint32_t failp = (r.flags >> AM_F_FAILP_SHIFT) & 0xFFu;
    const bool fail = (uint32_t)(k & 0xFF) < failp;
    const bool rem_ok = (uint32_t)((k >> 8) & 0xFF) < 179u;
    r.flags |= (fail ? AM_F_PENDING_FAIL : AM_F_PENDING_OK) | AM_F_REMEDY_PENDING | (rem_ok ? AM_F_REMEDY_OUTCOME_OK : 0u);
    act |= apply_result(r, T, res);
  }
  return act;
}

// The eight remedy / counter columns of record i, streamed in (flags and finishedAt are the caller's) ...
template <typename I>
__device__ __forceinline__ void load_state(const DevCols& c, I i, RecState& r) {
  r.limit = ld_stream(c.runs_limit + i); r.reset = ld_stream(c.reset_interval + i);
  r.s = ld_stream(c.success + i); r.f = ld_stream(c.failed + i);
  r.rs = ld_stream(c.remedy_success + i); r.rf = ld_stream(c.remedy_failed + i);
  r.rt = ld_stream(c.remedy_total + i); r.rfa = ld_stream(c.remedy_finished_at + i);
}
// ... and those of them that r changed against r0, streamed out
template <typename I>
__device__ __forceinline__ void store_changed_state(const DevCols& c, I i, const RecState& r, const RecState& r0) {
  if (r.s != r0.s) st_stream(c.success + i, r.s);
  if (r.f != r0.f) st_stream(c.failed + i, r.f);
  if (r.rs != r0.rs) st_stream(c.remedy_success + i, r.rs);
  if (r.rf != r0.rf) st_stream(c.remedy_failed + i, r.rf);
  if (r.rt != r0.rt) st_stream(c.remedy_total + i, r.rt);
  if (r.rfa != r0.rfa) st_stream(c.remedy_finished_at + i, r.rfa);
}

// The lanes' result counts (four 8-bit counts each, as apply_result adds them) summed over the warp: lane
// q < 4 gets counter q {ok, fail, remedy ok, remedy fail}.  Two redux over 16-bit halves; every lane calls it.
__device__ __forceinline__ uint32_t warp_result_count(uint32_t res, int lane) {
  uint32_t lo = 0, hi = 0;  // ok | fail << 16, remedy ok | remedy fail << 16
  if (__any_sync(kFull, res != 0)) { const uint2 s = warp_byte_sums(res); lo = s.x; hi = s.y; }
  return ((lane < 2 ? lo : hi) >> ((lane & 1) * 16)) & 0xFFFFu;
}

// kinds 1..5 are evaluated; tombstones, NO_RESOURCE (hcc.go:227) and host-fallback are not
__device__ __forceinline__ bool is_live(uint32_t f) { return ((0x3Eu >> (f & AM_KIND_MASK)) & 1u) && !(f & AM_F_TOMBSTONE); }
// INTERVAL or CRON_EVERY: due by the repeat timer
__device__ __forceinline__ bool is_interval_kind(uint32_t kind) { return ((0x14u >> kind) & 1u) != 0; }

// The interval rule, not(hcc.go:264): "elapsed < RepeatAfterSec && timer != nil" skips.  A posted result
// is applied first (step 1): finishedAt = T and the timer re-armed.  Without a timer (controller restart,
// hcc.go:161) the reference submits whatever finishedAt says.
__device__ __forceinline__ bool interval_due(uint32_t f, int32_t ras, int64_t fa, int64_t T) {
  const bool has_result = (f & kHcBits) != 0;
  const int64_t elapsed = (int64_t)((uint64_t)T - (uint64_t)(has_result ? T : fa));
  const bool armed = has_result || (f & AM_F_TIMER_ARMED) != 0;
  return !((elapsed < (int64_t)ras) & armed);
}

// The due word of a record against the handle's epoch E: its repeat deadline D = finishedAt + ras as an offset from
// E, clamped to [0, 0xFFFFFFFF].  For every T in [E, E + 0xFFFFFFFF) an armed record without a posted workflow phase is
// due (interval_due) exactly when T - E >= the word: D <= E gives 0 and T >= E >= D; D - E >= 0xFFFFFFFF gives the
// top word, which no T - E of the window reaches, and T < D.  Exact in the column domain (|time| < 2^55, i32 ras),
// where neither T - finishedAt nor finishedAt + ras overflows.  The DUE variants of the sweep read this word instead
// of ras and finishedAt; every writer of either column keeps it or the handle stops using it (sweep.cu, due_valid).
AM_HD uint32_t due_word(int32_t ras, int64_t fa, int64_t E) {
  const int64_t D = (int64_t)((uint64_t)fa + (uint64_t)(int64_t)ras);
  if (D <= E) return 0u;
  const uint64_t d = (uint64_t)D - (uint64_t)E;
  return d >= 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)d;
}
// The handle's epoch window: the seconds T whose T - E a due word decides.
constexpr int64_t kDueSpan = 0xFFFFFFFFll;
constexpr int64_t kDueEpochLead = 1ll << 31;  // a build at T takes E = T - 2^31: T sits in the middle of its window
// The sweep's use of the due words (sweep_tick_kernel's DUE): none, decide from them, or decide from ras and finishedAt
// as without them and write every swept record's word (the build, fused into an open-loop tick).
constexpr int kDueOff = 0, kDueRead = 1, kDueBuild = 2;

// The hold rule: the run in a since word is still in flight — it started no earlier than the record's finishedAt and
// no workflow phase is pending.  finishedAt and the flags are callables, read only when the terms before them hold.
template <typename FinishedAt, typename Flags>
__device__ __forceinline__ bool held_run(int64_t since, FinishedAt finished_at, Flags flags) {
  return since != kNotInFlight && since >= finished_at() && !(flags() & kHcBits);
}

// Action bits of apply_result <-> the carry bits of the flags word (AM_F_CARRY_MASK): RUN_REMEDY (0x02)
// in bit 11, REMEDY_SKIP .. ANOMALY (0x10 .. 0x80) in bits 12 .. 15.
__device__ __forceinline__ uint32_t carried_actions(uint32_t f) { return ((f >> 10) & AM_ACT_RUN_REMEDY) | ((f >> 8) & 0xF0u); }
__device__ __forceinline__ uint32_t carry_of_actions(uint32_t a) { return ((a & AM_ACT_RUN_REMEDY) << 10) | ((a & 0xF0u) << 8); }
static_assert(AM_F_CARRY_SHIFT == 11 && AM_ACT_RUN_REMEDY == 0x02u && AM_ACT_REMEDY_SKIP == 0x10u && AM_ACT_ANOMALY == 0x80u,
              "carry bit layout");

// Remedy hold: a result step whose actions `a` run the remedy starts a remedy run unless a remedy outcome (`f`, the flags
// it was applied to) completed the remedy at once.  In the reference the Failed branch blocks in watchRemedyWorkflow
// (hcc.go:683-714, :788-852) until the remedy ends; only then is the next run scheduled.
__device__ __forceinline__ bool starts_remedy_run(uint32_t a, uint32_t f) {
  return (a & AM_ACT_RUN_REMEDY) && !(f & AM_F_REMEDY_PENDING);
}
// The run of slot i started at T: since = T + kRemedyRun, and with timeout state (TIMEOUT) the deadline T + W of the
// slot's workflow timeout W (hcc.go:791-799 watch the remedy with Spec.Workflow.Timeout), none when W is 0 — stored
// either way, since the word may still hold the health-check run's deadline — and the segment's bound lowered to it.
// Starts are rare (a failure of a check with a remedy workflow): one atomic per start and no register kept live for it
// (a per-warp minimum cost the open-loop on-minute sweep 16 B of spills at 64 registers).
template <bool TIMEOUT>
__device__ __forceinline__ void start_remedy_run(int64_t* since, int64_t* deadline, const int32_t* wf_timeout,
                                                 unsigned long long* seg_deadline, uint32_t i, int64_t T) {
  since[i] = T + kRemedyRun;
  if (TIMEOUT) {
    const int32_t W = wf_timeout[i];
    deadline[i] = W > 0 ? T + W : kNoDeadline;
    if (W > 0) atomicMin(seg_deadline + i / (uint32_t)kRecPerWarp, biased_key(T + W));
  }
}

// robfig SpecSchedule matching against the tick's one-hot wall-clock words (Appendix A: five ANDs and
// the dom/dow star rule).  Branch-free: every term is evaluated (no short-circuit control flow).
__device__ __forceinline__ bool cron_matches(const TickWords& t, uint64_t mi, uint64_t hr, uint64_t dm, uint64_t mo, uint64_t dw) {
  const bool fld = ((mi & t.minute) != 0) & ((hr & t.hour) != 0) & ((mo & t.month) != 0);
  const bool dmm = (dm & t.dom) != 0, dwm = (dw & t.dow) != 0;
  const bool star = ((dm | dw) >> 63) != 0;  // robfig dayMatches
  return (t.sec0 != 0) & fld & (star ? (dmm & dwm) : (dmm | dwm));
}
// A schedule bound to a named time zone ("CRON_TZ=Zone ...", robfig parser.go / hcc.go:253,
// SpecSchedule.Location): the same match against the zone's wall clock.  `z` points at the zone's entry
// of the tick's word table (tz_words_kernel).  Rare records: kept out of line.  (Deriving the words from
// T + offset inside this call instead of loading them slowed the 10 M-record sweep — half of all warps
// hold a zone-bound record at 0.6 % of the records and ran ~100 more instructions each.)
__device__ __noinline__ bool cron_matches_in_zone(const TickWords* z, uint64_t mi, uint64_t hr, uint64_t dm, uint64_t mo,
                                                  uint64_t dw) {
  const TickWords t = *z;
  return cron_matches(t, mi, hr, dm, mo, dw);
}

// The tick's wall clock in every registered zone as one-hot words: T + the zone's UTC offset, broken
// down.  The offsets are kept by the launcher (valid until a zone changes its offset); this is one
// thread per zone and no memory traffic to speak of, launched with programmatic serialisation ahead of
// the sweep — only when zones are registered.
__global__ void tz_words_kernel(const int32_t* __restrict__ tz_off, TickWords* __restrict__ table, int64_t T, uint32_t n) {
  pdl_wait();
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) table[k] = tick_words_from_unix(T + (int64_t)tz_off[k]);
}

// ---------------------------------------------------------------------------
// The sweep.  CLOSED = closed-loop harness (SURVEY §8d config 5): a due record
// completes in the same tick with its preset outcome.
// ---------------------------------------------------------------------------
#ifndef AM_MIN_BLOCKS
#define AM_MIN_BLOCKS 3
#endif
// MASKS = the cron masks are read (as the six bit planes T tests) and matched.  Off
// the minute a 5-field schedule cannot fire (ParseStandard pins Second to 1<<0), so
// the launcher picks MASKS=false unless AM_SWEEP_FULL_SCAN is set: the plane loads
// and all of the mask arithmetic disappear at compile time.
// Registers: the closed-loop on-minute variant runs at AM_MIN_BLOCKS CTAs per SM (80 registers, 16 B of
// spill stores) and loads both halves' remedy state at once in its dense result path; the other three run
// at one more CTA per SM within 64 registers, one half at a time (the open-loop on-minute sweep measured
// faster so): the open-loop ones in 59 and 60 without spills, the closed-loop off-minute one with 20 B.
// WINDOW = a catch-up tick (AM_SWEEP_CATCH_UP, MASKS false): a 5-field schedule is due iff it fires somewhere in
// the window's calendar boxes (p.tz_table, per zone).  A box covers many values of a field, so no plane
// can answer it: the five canonical mask columns are read instead, 40 B per record, in warps that hold a
// CRON_SPEC record.  Runs at AM_MIN_BLOCKS CTAs per SM like the closed-loop on-minute variant.
// HOLD = hold in flight (am_sweep_set_hold_in_flight; open loop only): after the due decision, a due record whose
// health-check workflow is still running (held_run on p.since) is not
// submitted; every record that is submitted gets since = T.  The since word is loaded only for the halves that
// hold a due record: one dependent round trip, in the warps that have one (DESIGN.md section 3 compares it with
// streaming since for every record).
// TIMEOUT = workflow timeouts (HOLD only; the handle received a non-zero am_record_t.wf_timeout): the same round trip
// also loads the slot's timeout W, and every submitted record gets deadline = T + W (none when W is 0); one atomicMin
// per warp lowers the segment's bound (p.seg_deadline) that expire_runs_kernel reads.
// REMEDY = remedy hold (HOLD only, am_sweep_set_hold_remedy): a record whose posted result this sweep applies and which
// gains AM_ACT_RUN_REMEDY without a remedy outcome merged starts a remedy run (start_remedy_run): it is not submitted.
// DUE = kDueRead: the interval rule from the due words (open loop only, no window, no hold): phase A reads the 4-B word
// p.due instead of 4 B of ras and 8 B of finishedAt.  The few records whose decision or finishedAt needs more — a posted
// workflow phase (due iff ras <= 0, finishedAt = T) or STOPPED reported now (finishedAt = T) — load their ras on their
// own and store finishedAt and the new word one record at a time.  DUE = kDueBuild: the tick of DUE = kDueOff, which
// also writes every record's word from ras and the finishedAt the tick leaves.
template <bool CLOSED, bool MASKS, bool WINDOW = false, bool HOLD = false, bool TIMEOUT = false, bool REMEDY = false,
          int DUE = kDueOff>
__global__ void __launch_bounds__(kBlock, ((CLOSED && MASKS) || WINDOW) ? AM_MIN_BLOCKS : AM_MIN_BLOCKS + 1)
    sweep_tick_kernel(const SweepParams p) {
  // one row per warp, written unconditionally: no zero-initialisation, no shared
  // atomics, and therefore a single __syncthreads in the whole kernel
  __shared__ uint32_t s_warp_tot[kWarps], s_warp_exc[kWarps];
  __shared__ uint32_t s_ballot[kWarps][4];  // each warp's four emitted-record ballots
  __shared__ uint32_t s_wres[kWarps][4];    // posted results applied: ok, fail, remedy ok, remedy fail

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const uint32_t tile = blockIdx.x;
  const uint32_t tile_base = tile * (uint32_t)kTile;
  const int64_t T = p.T;
  pdl_wait();  // the sweep is launched while its predecessor (the previous tick's publish, or the drain) still runs
#ifdef AM_SWEEP_TRIGGER
  pdl_trigger();  // (A/B) scan_groups_kernel may become resident during the sweep's tail
#endif

  // ---- phase A: issue every schedule-column load of this lane up front ----
  // half h covers records r0(h) .. r0(h)+1, r0 = tile_base + warp*128 + h*64 + lane*2
  uint32_t r0[2];
  longlong2 fa[2];
  int2 ras[2];
  uint2 fl[2];
  uint2 dw[2];  // DUE: the due words
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    r0[h] = tile_base + (uint32_t)(warp * kRecPerWarp + h * 64 + lane * 2);
    fl[h] = ld_stream(reinterpret_cast<const uint2*>(p.c.flags + r0[h]));
    if (DUE == kDueRead) {
      dw[h] = ld_stream(reinterpret_cast<const uint2*>(p.due + r0[h]));
    } else {
      ras[h] = ld_stream(reinterpret_cast<const int2*>(p.c.ras + r0[h]));
      fa[h] = ld_stream(reinterpret_cast<const longlong2*>(p.c.finished_at + r0[h]));
    }
  }
  // The masks come from the six bit planes T tests (MaskPlanes): the warp's 128 records are 4 words of
  // each, one 16-B load per plane that every lane of the warp makes at the same address.  Nothing about
  // them depends on the flags.
  uint4 pmi, phr, pdm, pmo, pdw, pst;
  if (MASKS) {
    const uint32_t wq = (tile_base + (uint32_t)(warp * kRecPerWarp)) / 32u;
    pmi = ld_stream(reinterpret_cast<const uint4*>(p.pl.minute + wq));
    phr = ld_stream(reinterpret_cast<const uint4*>(p.pl.hour + wq));
    pdm = ld_stream(reinterpret_cast<const uint4*>(p.pl.dom + wq));
    pmo = ld_stream(reinterpret_cast<const uint4*>(p.pl.month + wq));
    pdw = ld_stream(reinterpret_cast<const uint4*>(p.pl.dow + wq));
    pst = ld_stream(reinterpret_cast<const uint4*>(p.pl.star + wq));
  }

  // Scheduling fence: a warp-level memory-ordering point.  ptxas may not sink the loads
  // above across it, so all of them are issued before any of the arithmetic below (without it
  // the second half's loads were delayed behind the first half's compute, at a large cost in bandwidth).
  __syncwarp();

  // The tick's broken-down time: one-hot words computed once per tick (civil.h) and
  // delivered through the kernel parameters, i.e. the constant bank / uniform
  // registers — cheaper than staging them in shared memory, which cost every CTA a
  // serial thread-0 section and a barrier.
  const TickWords w = p.words;
  // named time zones are rare: one vote per warp decides whether the per-record zone lookup exists at all
  const uint32_t fl_or = fl[0].x | fl[0].y | fl[1].x | fl[1].y;
  const bool warp_tz = MASKS && p.tz_table != nullptr && __any_sync(kFull, (fl_or >> AM_F_TZ_SHIFT) != 0);

  // cron_matches for 32 records per word: sec0 & MIN[m] & HR[h] & MO[mo] & dayMatches, where dayMatches
  // is DOM[d] & DOW[w] under the star bit S and DOM[d] | DOW[w] without it.  Word k of the segment holds
  // its records 32k .. 32k+31: the lane's records of half h are bits (2L & 31) + j of word 2h + (L >> 4).
  uint32_t cron_bits = 0;  // bit (2h+j): the record's 5-field schedule fires at T
  if (MASKS) {
    const uint32_t gate = w.sec0 ? kFull : 0u;
    auto word = [&](int k) {
      const uint32_t mi = k == 0 ? pmi.x : k == 1 ? pmi.y : k == 2 ? pmi.z : pmi.w;
      const uint32_t hr = k == 0 ? phr.x : k == 1 ? phr.y : k == 2 ? phr.z : phr.w;
      const uint32_t dm = k == 0 ? pdm.x : k == 1 ? pdm.y : k == 2 ? pdm.z : pdm.w;
      const uint32_t mo = k == 0 ? pmo.x : k == 1 ? pmo.y : k == 2 ? pmo.z : pmo.w;
      const uint32_t dw = k == 0 ? pdw.x : k == 1 ? pdw.y : k == 2 ? pdw.z : pdw.w;
      const uint32_t st = k == 0 ? pst.x : k == 1 ? pst.y : k == 2 ? pst.z : pst.w;
      return gate & mi & hr & mo & ((st & dm & dw) | (~st & (dm | dw)));
    };
    const uint32_t sh = (uint32_t)(2 * lane) & 31u;
#pragma unroll
    for (int h = 0; h < 2; ++h) cron_bits |= (((lane >> 4) ? word(2 * h + 1) : word(2 * h)) >> sh & 3u) << (2 * h);
    if (warp_tz) {  // warp-uniform: some record of this warp is bound to a named time zone
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint32_t f = j ? fl[h].y : fl[h].x;
          const uint32_t tz = f >> AM_F_TZ_SHIFT;
          // zone-bound records have no plane bits: their canonical masks against the zone's wall clock,
          // behind a real call (inlined, ptxas turned the zone lookup of all four records into predicated
          // instructions that EVERY warp issues: a clearly slower 10 M-record tick with 0.6 % zone-bound records)
          if (tz && (f & AM_KIND_MASK) == AM_KIND_CRON_SPEC) {
            const uint32_t i = r0[h] + (uint32_t)j;
            const bool m = cron_matches_in_zone(p.tz_table + tz, ld_stream(p.c.minute + i), ld_stream(p.c.hour + i),
                                                ld_stream(p.c.dom + i), ld_stream(p.c.month + i), ld_stream(p.c.dow + i));
            cron_bits |= (m ? 1u : 0u) << (2 * h + j);
          }
        }
      }
    }
  }
  if (WINDOW) {
    // one vote per warp: warps without a 5-field schedule read no masks
    uint32_t cron_lane = 0;  // bit (2h+j): the record is a CRON_SPEC one
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 2; ++j) cron_lane |= (((j ? fl[h].y : fl[h].x) & AM_KIND_MASK) == AM_KIND_CRON_SPEC ? 1u : 0u) << (2 * h + j);
    if (__any_sync(kFull, cron_lane != 0)) {
      ulonglong2 mi[2], hr[2], dm[2], mo[2], dw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mi[h] = ld_stream(reinterpret_cast<const ulonglong2*>(p.c.minute + r0[h]));
        hr[h] = ld_stream(reinterpret_cast<const ulonglong2*>(p.c.hour + r0[h]));
        dm[h] = ld_stream(reinterpret_cast<const ulonglong2*>(p.c.dom + r0[h]));
        mo[h] = ld_stream(reinterpret_cast<const ulonglong2*>(p.c.month + r0[h]));
        dw[h] = ld_stream(reinterpret_cast<const ulonglong2*>(p.c.dow + r0[h]));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((cron_lane >> (2 * h + j)) & 1u) {
            const TickWords* b = p.tz_table + ((j ? fl[h].y : fl[h].x) >> AM_F_TZ_SHIFT) * kWindowBoxes;
            bool m = false;
            for (int k = 0; k < kWindowBoxes && b[k].sec0; ++k)
              m |= cron_matches(b[k], j ? mi[h].y : mi[h].x, j ? hr[h].y : hr[h].x, j ? dm[h].y : dm[h].x,
                                j ? mo[h].y : mo[h].x, j ? dw[h].y : dw[h].x);
            cron_bits |= (m ? 1u : 0u) << (2 * h + j);
          }
        }
      }
    }
  }

  uint32_t act[2][2];
  uint32_t res_lane = 0;  // 4 x 8-bit counts of results applied by this lane
  uint32_t nfl[2][2];     // flags / finishedAt after this tick
  int64_t nfa[2][2];
  bool dirty[2] = {false, false};
  uint32_t needy = 0, due_bits = 0;  // bit (2h+j): record needs the remedy/counter columns / is due
  uint32_t fix = 0;                  // DUE, bit (2h+j): the tick sets the record's finishedAt to T

  // ---- schedule decision for the lane's four records ------------------------
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t f = j ? fl[h].y : fl[h].x;
      const int64_t fav = DUE == kDueRead ? 0 : (j ? fa[h].y : fa[h].x);
      const bool live = is_live(f);
      const bool pending = (f & kPendBits) != 0;
      // (an if, not `MASKS && ...`: with the latter ptxas hoisted this loop's arithmetic above the
      // __syncwarp fence in the MASKS=false variants and delayed the second half's loads behind it)
      bool due_cron = false;
      if (MASKS || WINDOW) due_cron = ((cron_bits >> (2 * h + j)) & 1u) != 0;
      const uint32_t kind = f & AM_KIND_MASK;
      bool due_iv;
      if (DUE == kDueRead)  // (a posted workflow phase: decided from ras below)
        due_iv = !(f & kHcBits) && (!(f & AM_F_TIMER_ARMED) || p.due_t >= (j ? dw[h].y : dw[h].x));
      else
        due_iv = interval_due(f, j ? ras[h].y : ras[h].x, fav, T);
      const bool is_iv = is_interval_kind(kind);
      // (the rest of the ladder is written out here and in block_record: behind a function, ptxas turned
      // these `live && ...` into branch-free code that spilled more in the closed-loop on-minute variant)
      const bool due = live && (is_iv ? due_iv : (kind == AM_KIND_CRON_SPEC && due_cron));
      const bool stopped_now = live && kind == AM_KIND_STOPPED && !(f & AM_F_STOPPED_REPORTED);
      act[h][j] = (due ? AM_ACT_SUBMIT_HC : 0u) | (stopped_now ? AM_ACT_STOPPED : 0u) |
                  ((live && kind == AM_KIND_PARSE_ERROR) ? AM_ACT_PARSE_ERROR : 0u);
      nfl[h][j] = f;
      nfa[h][j] = fav;
      if (stopped_now) {  // hcc.go:238-250: Status "Stopped", FinishedAt = now
        nfl[h][j] = f | AM_F_STOPPED_REPORTED;
        nfa[h][j] = T;
        dirty[h] = true;
      }
      if (live && (pending || (CLOSED && due))) needy |= 1u << (2 * h + j);
      if (due) due_bits |= 1u << (2 * h + j);
      if (DUE && live && (stopped_now || (f & kHcBits))) fix |= 1u << (2 * h + j);
    }
  }

  // ---- kDueBuild: every record's word, from its finishedAt after this tick (T where `fix` says so)
  if (DUE == kDueBuild) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t a0 = (fix >> (2 * h)) & 1u ? T : fa[h].x, a1 = (fix >> (2 * h + 1)) & 1u ? T : fa[h].y;
      st_stream(reinterpret_cast<uint2*>(p.due + r0[h]),
                make_uint2(due_word(ras[h].x, a0, p.due_epoch), due_word(ras[h].y, a1, p.due_epoch)));
    }
  }
  // ---- kDueRead: the records whose finishedAt this tick sets to T (apply_result does for a workflow phase, and the
  //      pause rule for STOPPED; both when the two meet).  Rare: their ras one record at a time, which also decides a
  //      posted phase's interval rule (elapsed 0: due iff ras <= 0), then finishedAt and the new due word.
  if (DUE == kDueRead && __any_sync(kFull, fix != 0)) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if ((fix >> q) & 1u) {
        const uint32_t i = r0[q >> 1] + (uint32_t)(q & 1);
        const uint32_t f = (q & 1) ? fl[q >> 1].y : fl[q >> 1].x;
        const int32_t rv = ld_stream(p.c.ras + i);
        if ((f & kHcBits) && is_interval_kind(f & AM_KIND_MASK) && rv <= 0) act[q >> 1][q & 1] |= AM_ACT_SUBMIT_HC;
        st_stream(p.c.finished_at + i, T);
        st_stream(p.due + i, due_word(rv, T, p.due_epoch));
      }
    }
  }

  // ---- hold in flight: the reference's watch loop holds a check until its workflow ends (hcc.go:607-727) and only
  //      then arms the next timer (hcc.go:745-752).  A posted phase clears since at the drain (clear_since_kernel).
  if (HOLD && __any_sync(kFull, due_bits != 0)) {
    unsigned long long dmin = ~0ull;  // TIMEOUT: the least deadline this lane set (biased key)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t db = (due_bits >> (2 * h)) & 3u;
      if (db) {
        const longlong2 sv = ld_stream(reinterpret_cast<const longlong2*>(p.since + r0[h]));
        int2 wv = make_int2(0, 0);
        if (TIMEOUT) wv = ld_stream(reinterpret_cast<const int2*>(p.wf_timeout + r0[h]));
        int64_t s[2] = {sv.x, sv.y};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((db >> j) & 1u) {
            const uint32_t f = j ? fl[h].y : fl[h].x;
            const int64_t fav = j ? fa[h].y : fa[h].x;
            // held_run, written out: through the call the hold variants compile to different machine code
            if (s[j] != kNotInFlight && s[j] >= fav && !(f & kHcBits)) {
              act[h][j] &= ~AM_ACT_SUBMIT_HC;
            } else {
              s[j] = T;
              if (TIMEOUT) {  // the run's deadline is fixed at its submission (hcc.go:611-613); a new run replaces it
                const int32_t W = j ? wv.y : wv.x;
                const int64_t D = W > 0 ? T + W : kNoDeadline;
                st_stream(p.deadline + r0[h] + j, D);
                if (W > 0 && biased_key(D) < dmin) dmin = biased_key(D);
              }
            }
          }
        }
        if (s[0] != sv.x || s[1] != sv.y) st_stream(reinterpret_cast<longlong2*>(p.since + r0[h]), make_longlong2(s[0], s[1]));
      }
    }
    if (TIMEOUT && __any_sync(kFull, dmin != ~0ull)) {  // one atomic per warp into its segment's bound
      dmin = warp_min(dmin);
      if (lane == 0) atomicMin(p.seg_deadline + (tile_base + (uint32_t)(warp * kRecPerWarp)) / (uint32_t)kRecPerWarp, dmin);
    }
  }

  // ---- results applied at this tick's drain (apply_results_now_kernel) left their action bits in the
  //      flags' carry bits: emit and clear them.  Rare (a posted "Succeeded" carries nothing): one vote
  //      per warp keeps the per-record form out of the common path.
  if (__any_sync(kFull, (fl_or & AM_F_CARRY_MASK) != 0)) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint32_t f = j ? fl[h].y : fl[h].x;
        if (f & AM_F_CARRY_MASK) {
          act[h][j] |= carried_actions(f);
          nfl[h][j] &= ~AM_F_CARRY_MASK;
          dirty[h] = true;
        }
      }
    }
  }

  // ---- results + remedy state machine (hcc.go:633-724, 819-852) -------------------
  // Two shapes, chosen per warp by how many lanes have work:
  //  dense  (>= 16 lanes, e.g. half of all checks reporting a result this tick): per
  //         pair of records, vector loads of the eight remedy/counter columns and the
  //         state machine predicated per record — the bytes are needed anyway and 16-B
  //         transactions keep the LSU count low;
  //  sparse (a few due/posted records per warp): a warp loop in which every lane takes
  //         its next needy record with scalar accesses — the loop runs once or twice
  //         instead of four predicated copies of the state machine.
  if (__popc(__ballot_sync(kFull, needy != 0)) >= 16) {
    // at 80 registers both halves' loads first (sixteen more in flight per lane),
    // then the state machines, then the stores — a half's stores would otherwise fence the other
    // half's loads behind them (the compiler cannot tell the columns apart)
    int2 lim[2], rst[2], sc[2], fc[2], rsc[2], rfc[2], rtc[2];
    longlong2 rfa[2];
    auto load_half = [&](int h) {
      if ((needy >> (2 * h)) & 3u) {
        const uint32_t r = r0[h];
        lim[h] = ld_stream(reinterpret_cast<const int2*>(p.c.runs_limit + r));
        rst[h] = ld_stream(reinterpret_cast<const int2*>(p.c.reset_interval + r));
        sc[h] = ld_stream(reinterpret_cast<const int2*>(p.c.success + r));
        fc[h] = ld_stream(reinterpret_cast<const int2*>(p.c.failed + r));
        rsc[h] = ld_stream(reinterpret_cast<const int2*>(p.c.remedy_success + r));
        rfc[h] = ld_stream(reinterpret_cast<const int2*>(p.c.remedy_failed + r));
        rtc[h] = ld_stream(reinterpret_cast<const int2*>(p.c.remedy_total + r));
        rfa[h] = ld_stream(reinterpret_cast<const longlong2*>(p.c.remedy_finished_at + r));
      }
    };
    if (CLOSED && (MASKS || WINDOW)) {  // (the variants at 64 registers: one half at a time)
      load_half(0);
      load_half(1);
      __syncwarp();
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t nb = (needy >> (2 * h)) & 3u;
      if (!(CLOSED && (MASKS || WINDOW))) load_half(h);
      if (nb) {
        const uint32_t r = r0[h];
        int32_t ns[2] = {sc[h].x, sc[h].y}, nf[2] = {fc[h].x, fc[h].y};
        int32_t nrs[2] = {rsc[h].x, rsc[h].y}, nrf[2] = {rfc[h].x, rfc[h].y}, nrt[2] = {rtc[h].x, rtc[h].y};
        int64_t nrfa[2] = {rfa[h].x, rfa[h].y};
        const int32_t limv[2] = {lim[h].x, lim[h].y}, rstv[2] = {rst[h].x, rst[h].y};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((nb >> j) & 1u) {
            RecState s{nfl[h][j], nfa[h][j], ns[j], nf[j], nrs[j], nrf[j], nrt[j], nrfa[j], limv[j], rstv[j]};
            uint32_t res = 0;
            const uint32_t a = result_step<CLOSED>(s, T, (due_bits >> (2 * h + j)) & 1u, p.seed, p.shard_base + r + (uint32_t)j, res);
            act[h][j] |= a;
            if (REMEDY && starts_remedy_run(a, nfl[h][j])) {
              start_remedy_run<TIMEOUT>(p.since, p.deadline, p.wf_timeout, p.seg_deadline, r + (uint32_t)j, T);
              act[h][j] &= ~AM_ACT_SUBMIT_HC;
            }
            res_lane += res;
            nfl[h][j] = s.flags; nfa[h][j] = s.fa;
            ns[j] = s.s; nf[j] = s.f; nrs[j] = s.rs; nrf[j] = s.rf; nrt[j] = s.rt; nrfa[j] = s.rfa;
          }
        }
        dirty[h] = true;  // a result always clears its PENDING flags
        if (ns[0] != sc[h].x || ns[1] != sc[h].y) st_stream(reinterpret_cast<int2*>(p.c.success + r), make_int2(ns[0], ns[1]));
        if (nf[0] != fc[h].x || nf[1] != fc[h].y) st_stream(reinterpret_cast<int2*>(p.c.failed + r), make_int2(nf[0], nf[1]));
        if (nrs[0] != rsc[h].x || nrs[1] != rsc[h].y)
          st_stream(reinterpret_cast<int2*>(p.c.remedy_success + r), make_int2(nrs[0], nrs[1]));
        if (nrf[0] != rfc[h].x || nrf[1] != rfc[h].y)
          st_stream(reinterpret_cast<int2*>(p.c.remedy_failed + r), make_int2(nrf[0], nrf[1]));
        if (nrt[0] != rtc[h].x || nrt[1] != rtc[h].y)
          st_stream(reinterpret_cast<int2*>(p.c.remedy_total + r), make_int2(nrt[0], nrt[1]));
        if (nrfa[0] != rfa[h].x || nrfa[1] != rfa[h].y)
          st_stream(reinterpret_cast<longlong2*>(p.c.remedy_finished_at + r), make_longlong2(nrfa[0], nrfa[1]));
      }
    }
    needy = 0;
  }
  while (__any_sync(kFull, needy != 0)) {
    if (needy) {
      const int b = __ffs(needy) - 1;
      needy &= needy - 1;
      const uint32_t i = r0[0] + (uint32_t)(64 * (b >> 1) + (b & 1));
      RecState s;
      load_state(p.c, i, s);
      s.flags = b == 0 ? nfl[0][0] : b == 1 ? nfl[0][1] : b == 2 ? nfl[1][0] : nfl[1][1];
      s.fa = b == 0 ? nfa[0][0] : b == 1 ? nfa[0][1] : b == 2 ? nfa[1][0] : nfa[1][1];
      const RecState s0 = s;
      uint32_t res = 0;
      const uint32_t a = result_step<CLOSED>(s, T, (due_bits >> b) & 1u, p.seed, p.shard_base + i, res);
      res_lane += res;  // per lane at most 4 records x 2 results per byte
      store_changed_state(p.c, i, s, s0);
      const bool run = REMEDY && starts_remedy_run(a, s0.flags);
      if (run) start_remedy_run<TIMEOUT>(p.since, p.deadline, p.wf_timeout, p.seg_deadline, i, T);
      // (a record "Stopped" in this very tick already carries STOPPED_REPORTED and
      // finishedAt = T in nfl/nfa, and apply_result preserves both: the pause rule of
      // hcc.go:238-250 and a posted result commute)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q == b) {
          act[q >> 1][q & 1] |= a;
          if (run) act[q >> 1][q & 1] &= ~AM_ACT_SUBMIT_HC;
          nfl[q >> 1][q & 1] = s.flags;
          nfa[q >> 1][q & 1] = s.fa;
        }
      }
      if (b < 2) dirty[0] = true; else dirty[1] = true;  // a result always clears its PENDING flags
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (dirty[h]) {
      st_stream(reinterpret_cast<uint2*>(p.c.flags + r0[h]), make_uint2(nfl[h][0], nfl[h][1]));
      if (DUE != kDueRead)  // (kDueRead: stored above, per record)
        st_stream(reinterpret_cast<longlong2*>(p.c.finished_at + r0[h]), make_longlong2(nfa[h][0], nfa[h][1]));
    }
  }

  // ---- the emitted set as a bitmap, non-default actions as exceptions -------------
  // e..: records with any action; x..: records whose action is not the bare SUBMIT_HC (rare
  // unless results are being applied: their ballots are only taken when the warp has any)
  const unsigned e00 = __ballot_sync(kFull, act[0][0] != 0), e01 = __ballot_sync(kFull, act[0][1] != 0);
  const unsigned e10 = __ballot_sync(kFull, act[1][0] != 0), e11 = __ballot_sync(kFull, act[1][1] != 0);
  const uint32_t warp_total = __popc(e00) + __popc(e01) + __popc(e10) + __popc(e11);
  unsigned x00 = 0, x01 = 0, x10 = 0, x11 = 0;
  if (__any_sync(kFull, (act[0][0] | act[0][1] | act[1][0] | act[1][1]) > 1u)) {
    x00 = __ballot_sync(kFull, act[0][0] > 1u); x01 = __ballot_sync(kFull, act[0][1] > 1u);
    x10 = __ballot_sync(kFull, act[1][0] > 1u); x11 = __ballot_sync(kFull, act[1][1] > 1u);
  }
  const uint32_t xtot0 = __popc(x00) + __popc(x01);
  const uint32_t warp_exc = xtot0 + __popc(x10) + __popc(x11);
  // the four ballots go to shared memory as they are; warp 0 interleaves them into the tile's 32
  // bitmap words after the barrier (once per tile instead of once per warp)
  if (lane < 4) s_ballot[warp][lane] = lane == 0 ? e00 : (lane == 1 ? e01 : (lane == 2 ? e10 : e11));
  if (lane == 0) { s_warp_tot[warp] = warp_total; s_warp_exc[warp] = warp_exc; }

  // ---- results applied this tick (feeds metrics.MonitorSuccess/Error): lane ->
  //      warp -> per-warp shared row.  The action statistics and index checksums are
  //      derived from the emitted entries by expand_kernel, so records that emit
  //      nothing cost nothing here.
  {
    const uint32_t v = warp_result_count(res_lane, lane);
    if (lane < 4) s_wres[warp][lane] = v;
  }
  __syncthreads();

  // ---- tile write-out: one 128-B line of bitmap words, the counts, the exceptions ---
  // Everything written here is read once, a few tens of microseconds later, by
  // expand_kernel (and by the NVLink push): keep it L2-resident (evict_last) while the
  // evict_first column data streams past.
  const uint64_t keep = l2_evict_last_policy();
  if (warp == 0) {
    // Word `lane` of the tile = word k = lane & 3 of warp lane >> 2: its records 32k .. 32k+31 are
    // half k>>1, lanes 16(k&1) .. +15, two records per lane — the two ballots of that half, 16
    // bits each, interleaved.
    const int ww = lane >> 2, hh = (lane >> 1) & 1;
    const unsigned sh16 = (unsigned)(lane & 1) * 16u;
    const uint32_t word = spread16(s_ballot[ww][2 * hh] >> sh16) | (spread16(s_ballot[ww][2 * hh + 1] >> sh16) << 1);
    st_keep_u32(p.out.bitmap + (size_t)tile * kTileWords + lane, word, keep);
    if (lane < 4) {  // result counters (RED, no return value)
      uint32_t sv = 0;
#pragma unroll
      for (int k = 0; k < kWarps; ++k) sv += s_wres[k][lane];
      if (sv) atomicAdd(&p.acc[10 + lane], (unsigned long long)sv);
    }
    if (lane == 4 || lane == 5) {
      uint32_t tot = 0;
#pragma unroll
      for (int k = 0; k < kWarps; ++k) tot += lane == 4 ? s_warp_tot[k] : s_warp_exc[k];
      if (lane == 4) { if (tot) atomicAdd(&p.out.group_count[tile / kGroupTiles], tot); }
      else st_keep_u32(p.out.tile_exc + tile, tot, keep);
    }
  }
  if (warp_exc) {  // warp-uniform; rare unless results are being applied
    uint32_t base = tile_base;
#pragma unroll
    for (int k = 0; k < kWarps; ++k) base += (k < warp) ? s_warp_exc[k] : 0u;
    const unsigned lt = (1u << lane) - 1u;
    uint32_t rank[2];
    rank[0] = __popc(x00 & lt) + __popc(x01 & lt);
    rank[1] = xtot0 + __popc(x10 & lt) + __popc(x11 & lt);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t pos = base + rank[h];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (act[h][j] > 1u) {
          const uint32_t off = (uint32_t)(warp * kRecPerWarp + h * 64 + lane * 2 + j);  // record within the tile
          st_keep_u32(p.out.exc_seg + pos, exc_entry(off, act[h][j]), keep);
          ++pos;
        }
    }
  }
}

// ---------------------------------------------------------------------------
// Per-group emitted counts -> exclusive offsets.  One CTA: the array is a few KB (one u32
// per 8192 records; 1221 for 10 M records) and the work is O(groups) whatever the shard size
// — round 1 had every compaction CTA re-sum all earlier groups, O(groups^2) loads per tick.
// Also publishes n_emitted early (acc[1], and min(n_emitted, cap) for device-side consumers
// of the list) and zeroes the group counters again for the next tick.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) scan_groups_kernel(const ScanParams p) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  pdl_wait();  // the sweep's REDs into group_count are complete and visible
  pdl_trigger();
  __syncthreads();
  for (uint32_t g0 = 0; g0 < p.n_groups; g0 += blockDim.x) {
    const uint32_t g = g0 + (uint32_t)tid;
    const uint32_t c = g < p.n_groups ? p.group_count[g] : 0u;
    const uint32_t incl = warp_inclusive_scan(c, lane);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the 32 warp totals
      const uint32_t t = s_warp[lane];
      s_warp[lane] = warp_inclusive_scan(t, lane) - t;
    }
    __syncthreads();
    const uint32_t carry = s_carry;
    const uint32_t excl = carry + s_warp[warp] + incl - c;
    if (g < p.n_groups) {
      p.group_prefix[g] = excl;
      p.group_count[g] = 0;  // re-armed for the next tick that uses this buffer set
    }
    __syncthreads();  // every thread has read s_carry / s_warp of this round
    if (tid == (int)blockDim.x - 1) s_carry = excl + c;
    __syncthreads();
  }
  if (tid == 0) {
    const uint32_t total = s_carry;
    p.group_prefix[p.n_groups] = total;
    p.acc[1] = (unsigned long long)total;  // n_emitted
    if (p.out_count) *p.out_count = total < p.cap ? total : p.cap;
  }
}

// ---------------------------------------------------------------------------
// Bitmap + exceptions -> the contiguous ascending (index, action) list.  One CTA per
// (group, rank): thread t owns bitmap words 2t, 2t+1 of the group (64 records).  The CTA's position
// in the output is rank offset + group_prefix[g]; the in-group rank of a set bit is the
// exclusive popcount prefix of its word (warp shuffles + 4 warp totals) plus the bits below
// it.  Offsets and action bytes are staged in shared memory — defaults first, then the
// tile's exceptions patched in by rank lookup — and written out as destination-aligned
// quads (16 B of indices + 4 B of actions per store), so the same kernel can write into
// HBM, into a peer-visible exchange buffer or straight into mapped host memory.  While
// writing, every thread counts action bits and checksums global indices for the shard
// whose statistics this GPU owns.
// ---------------------------------------------------------------------------
constexpr int kExpandThreads = 128;  // one thread per PAIR of bitmap words (64 records): the kernel is
                                     // instruction-bound, and the per-thread fixed cost halves per entry
__global__ void __launch_bounds__(kExpandThreads, 8) expand_kernel(const ExpandParams p) {
  // staged so that shared index j <-> output position (start & ~3) + j: a destination-aligned
  // quad of the output is one aligned 8-B (offsets) + one 4-B (actions) shared load
  __shared__ __align__(16) uint16_t s_off[kGroupRecords + 8];
  __shared__ __align__(16) uint8_t s_act[kGroupRecords + 8];
  __shared__ uint32_t s_w[kGroupWords];
  __shared__ uint16_t s_wpre[kGroupWords];
  __shared__ uint32_t s_warp[4];
  __shared__ uint32_t s_nx[8];
  __shared__ uint32_t s_cnt[4][8];            // per-warp counts of the 8 action bits among the exceptions
  __shared__ unsigned long long s_chk[4][2];  // per-warp xor / sum of emitted global indices
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r = blockIdx.y;
  const uint32_t g = blockIdx.x;
  const ExpandSrc& src = p.src[r];
  if (g >= src.n_groups) return;  // uniform per CTA
  pdl_wait();
  pdl_trigger();
  // ---- every global load of the CTA is issued here, before the first use: the kernel is a chain
  //      of L2 latencies otherwise (one CTA moves 1 KB in and ~14 KB out)
  const uint2 w2 = __ldcs(reinterpret_cast<const uint2*>(src.bitmap + (size_t)g * kGroupWords) + tid);
  uint64_t start = src.group_prefix[g];
  const uint32_t cnt = src.group_prefix[g + 1] - (uint32_t)start;
  // Exceptions: half-warp (tile & 1) of warp (tile >> 1) patches tile `tile` of the group; its first
  // 16 entries are fetched speculatively (the segment is always mapped; entries past the count are
  // never used)
  const uint32_t tsub = (uint32_t)tid >> 4, l16 = (uint32_t)tid & 15u;  // tile within the group, lane within the half-warp
  const uint32_t tile = g * kGroupTiles + tsub;
  const bool tile_ok = tile < src.n_tiles;
  const uint32_t nx = tile_ok ? src.tile_exc[tile] : 0u;
  const uint32_t e_first = tile_ok ? __ldcs(src.exc_seg + (size_t)tile * kTile + l16) : 0u;
  for (int q = 0; q < r; ++q) start += p.src[q].group_prefix[p.src[q].n_groups];
  if (cnt == 0) return;  // uniform per CTA: nothing emitted by these 8192 records
  const uint32_t sh = (uint32_t)start & 3u;

  // ---- ranks: exclusive popcount prefix over the group's 256 words (two per thread)
  const uint32_t c_lo = (uint32_t)__popc(w2.x), c = c_lo + (uint32_t)__popc(w2.y);
  const uint32_t incl = warp_inclusive_scan(c, lane);
  if (lane == 31) s_warp[warp] = incl;
  if (l16 == 0) s_nx[tsub] = nx;
  *reinterpret_cast<uint2*>(&s_w[2 * tid]) = w2;
  // default action for every staged entry (and the padding around them), 4 bytes per store
  for (uint32_t j = (uint32_t)tid * 4u; j < sh + cnt + 4u; j += 4u * kExpandThreads)
    *reinterpret_cast<uint32_t*>(&s_act[j]) = 0x01010101u * AM_ACT_SUBMIT_HC;
  __syncthreads();
  uint32_t before = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) before += k < warp ? s_warp[k] : 0u;
  const uint32_t excl = before + incl - c;
  *reinterpret_cast<uint32_t*>(&s_wpre[2 * tid]) = excl | ((excl + c_lo) << 16);
  {  // two 32-bit loops (a 64-bit find-first-set / clear-lowest pair costs twice the instructions)
    uint32_t pos = sh + excl;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      uint32_t ww = hf ? w2.y : w2.x;
      const uint32_t rec0 = (uint32_t)tid * 64u + (uint32_t)hf * 32u - 1u;  // __ffs is 1-based
      while (ww) {
        s_off[pos++] = (uint16_t)(rec0 + (uint32_t)__ffs((int)ww));
        ww &= ww - 1u;
      }
    }
  }
  __syncthreads();
  // ---- exceptions of this half-warp's tile: action bytes other than the default.  Their action
  //      bits are counted here (the default entries all carry SUBMIT_HC and nothing else).
  const bool stats = p.acc != nullptr && r == p.stats_rank;
  uint32_t c0 = 0, c1 = 0;
  for (uint32_t i = l16; i < nx; i += 16u) {
    const uint32_t e = i < 16u ? e_first : __ldcs(src.exc_seg + (size_t)tile * kTile + i);
    const uint32_t off = tsub * (uint32_t)kTile + exc_offset(e), a = exc_action(e);
    const uint32_t wd = off >> 5;
    const uint32_t rk = (uint32_t)s_wpre[wd] + (uint32_t)__popc(s_w[wd] & ((1u << (off & 31u)) - 1u));
    s_act[sh + rk] = (uint8_t)a;
    c0 += spread4(a);
    c1 += spread4(e >> 4);  // the action's high nibble (spread4 reads 4 bits: masking a first costs instructions)
  }
  if (stats) {
    // statistics of this warp's slice of the group: action bits from the exceptions (a lane holds
    // at most 64 of them: byte counters), index checksums from the bitmap words themselves — the
    // sum over the set bits b of word t of (32 t + b) = popc(w) 32 t + sum_j 2^j popc(w & M_j)
    uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;  // action bits 0 | 1 << 16, ..., 6 | 7 << 16
    if (__any_sync(kFull, nx != 0)) {
      const uint2 s0 = warp_byte_sums(c0), s1 = warp_byte_sums(c1);
      a0 = s0.x; a1 = s0.y; a2 = s1.x; a3 = s1.y;
    }
    if (lane < 8) {
      const uint32_t qv = lane < 2 ? a0 : (lane < 4 ? a1 : (lane < 6 ? a2 : a3));
      s_cnt[warp][lane] = (qv >> ((lane & 1) * 16)) & 0xFFFFu;
    }
    uint32_t osum = 0;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const uint32_t w = hf ? w2.y : w2.x;
      osum += (uint32_t)__popc(w) * ((uint32_t)(2 * tid + hf) * 32u) + (uint32_t)__popc(w & 0xAAAAAAAAu) +
              2u * (uint32_t)__popc(w & 0xCCCCCCCCu) + 4u * (uint32_t)__popc(w & 0xF0F0F0F0u) +
              8u * (uint32_t)__popc(w & 0xFF00FF00u) + 16u * (uint32_t)__popc(w & 0xFFFF0000u);
    }
    const uint32_t wsum = __reduce_add_sync(kFull, osum);  // < 2^25 per warp
    if (lane == 0) s_chk[warp][1] = wsum;
  }
  __syncthreads();

  // ---- write-out: destination-aligned quads
  const uint64_t obase = src.base + (uint64_t)g * kGroupRecords;
  const uint64_t sbase = p.stats_base + (uint64_t)g * kGroupRecords;
  const uint64_t pos_base = start - sh;  // multiple of 4
  const uint32_t n_stage = sh + cnt;
  unsigned long long cx = 0;
  // any quad, entry by entry: the ragged first / last quad of the group, the end of a short buffer
  auto write_ragged = [&](uint32_t j) {
    const uint2 o2 = *reinterpret_cast<const uint2*>(&s_off[4u * j]);
    const uint32_t a4 = *reinterpret_cast<const uint32_t*>(&s_act[4u * j]);
    const uint32_t off[4] = {o2.x & 0xFFFFu, o2.x >> 16, o2.y & 0xFFFFu, o2.y >> 16};
    const uint64_t pos0 = pos_base + 4ull * j;
    const uint32_t k_lo = j == 0 ? sh : 0u;
    const uint32_t k_hi = n_stage - 4u * j < 4u ? n_stage - 4u * j : 4u;
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
      if (k < k_lo || k >= k_hi) continue;
      if (stats) cx ^= sbase + off[k];
      const uint64_t pos = pos0 + k;
      if (pos >= p.cap) continue;
      if (p.idx_bytes == 4) reinterpret_cast<uint32_t*>(p.out_idx)[pos] = (uint32_t)(obase + off[k]);
      else reinterpret_cast<uint64_t*>(p.out_idx)[pos] = obase + off[k];
      p.out_act[pos] = (uint8_t)(a4 >> (8 * k));
    }
  };
  // Interior quads [q_lo, q_hi): all four slots belong to this group and fit the caller's buffer — no
  // per-entry predicates (they were two thirds of this loop's 71 instructions per quad).  The index
  // checksum runs on the low words: a group's indices share their high word unless the group straddles
  // a multiple of 2^32 (then every quad takes the entry-by-entry form), and four equal high words cancel.
  const uint32_t q_lo = sh ? 1u : 0u;
  uint32_t q_hi = n_stage >> 2;
  {
    const uint64_t cap_q = p.cap >> 2, base_q = pos_base >> 2;
    const uint64_t room = cap_q > base_q ? cap_q - base_q : 0;
    if (room < q_hi) q_hi = (uint32_t)room;
    if ((uint32_t)sbase > 0xFFFFFFFFu - kGroupRecords) q_hi = q_lo;  // (uniform per CTA)
    if (q_hi < q_lo) q_hi = q_lo;
  }
  const uint32_t n_quads = (n_stage + 3u) >> 2;
  if (q_lo && (uint32_t)tid == 0u) write_ragged(0);
  for (uint32_t j = q_hi + (uint32_t)tid; j < n_quads; j += blockDim.x) write_ragged(j);
  {
    const uint32_t b32 = (uint32_t)obase, s32 = (uint32_t)sbase;
    uint32_t cx32 = 0;
    for (uint32_t j = q_lo + (uint32_t)tid; j < q_hi; j += blockDim.x) {
      const uint2 o2 = *reinterpret_cast<const uint2*>(&s_off[4u * j]);
      const uint32_t a4 = *reinterpret_cast<const uint32_t*>(&s_act[4u * j]);
      const uint32_t o0 = o2.x & 0xFFFFu, o1 = o2.x >> 16, o2_ = o2.y & 0xFFFFu, o3 = o2.y >> 16;
      const uint64_t q = (pos_base >> 2) + j;
      if (p.idx_bytes == 4) {
        reinterpret_cast<uint4*>(p.out_idx)[q] = make_uint4(b32 + o0, b32 + o1, b32 + o2_, b32 + o3);
      } else {
        ulonglong2* d = reinterpret_cast<ulonglong2*>(p.out_idx) + 2 * q;
        d[0] = make_ulonglong2(obase + o0, obase + o1);
        d[1] = make_ulonglong2(obase + o2_, obase + o3);
      }
      reinterpret_cast<uint32_t*>(p.out_act)[q] = a4;
      cx32 ^= (s32 + o0) ^ (s32 + o1) ^ (s32 + o2_) ^ (s32 + o3);
    }
    if (stats) cx ^= (unsigned long long)cx32;
  }
  // statistics: warp -> CTA -> global RED
  if (stats) {
    const uint32_t xl = __reduce_xor_sync(kFull, (uint32_t)cx), xh = __reduce_xor_sync(kFull, (uint32_t)(cx >> 32));
    if (lane == 0) s_chk[warp][0] = ((unsigned long long)xh << 32) | xl;
    __syncthreads();
    if (tid < 8) {
      uint32_t v = 0, n_exc = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) v += s_cnt[k][tid];
#pragma unroll
      for (int k = 0; k < 8; ++k) n_exc += s_nx[k];
      if (tid == 0) v += cnt - n_exc;  // every default entry is a bare SUBMIT_HC
      if (v) atomicAdd(&p.acc[2 + tid], (unsigned long long)v);
    }
    if (tid == 8) {
      unsigned long long x = 0, t = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) { x ^= s_chk[k][0]; t += s_chk[k][1]; }
      atomicXor(&p.acc[14], x);
      atomicAdd(&p.acc[15], t + (unsigned long long)cnt * sbase);
    }
  }
}

// One warp, after the kernel boundary that completes every expand CTA's REDs: publish the
// tick's am_tick_stats_t (device or mapped-host memory) and re-arm the accumulators.
__global__ void publish_kernel(unsigned long long* acc, am_tick_stats_t* out_stats, uint64_t n_records) {
  const int k = threadIdx.x;
  if (k >= kNumAcc) return;
  pdl_wait();
  unsigned long long v = acc[k];
  acc[k] = 0;
  if (k == 0) v = n_records;
  if (out_stats) reinterpret_cast<unsigned long long*>(out_stats)[k] = v;
}

// ---- small maintenance kernels (create / read) -----------------------------
__global__ void fill_u32_kernel(uint32_t* p, uint32_t v, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// RepeatAfterSec as the reference derives it at reconcile time (hcc.go:259-262):
// for a 5-field schedule Next(T) - T (robfig SpecSchedule.Next, cron_next_utc), for
// "@every d" and interval checks the stored interval, 0 for everything else.  One
// thread per record; the day scan diverges, which is fine for an on-demand query
// (status display, timer-wheel bucketing) that is not part of the per-tick path.
// A schedule bound to a named time zone is written as kZoneBoundMark: the host evaluates its Next()
// (am_cron_next).  No answer takes that value: a 5-field schedule's is > 0 or -9223372035 (|T| < 2^55),
// an interval's is an i32, whatever its sign.
constexpr int64_t kZoneBoundMark = INT64_MIN;

__global__ void next_fire_kernel(DevCols c, uint32_t first, uint32_t n, int64_t T, int64_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = first + k;
  const uint32_t f = c.flags[i];
  const uint32_t kind = f & AM_KIND_MASK;
  int64_t v = 0;
  if (!(f & AM_F_TOMBSTONE)) {
    if (kind == AM_KIND_CRON_SPEC && (f >> AM_F_TZ_SHIFT) != 0)
      v = kZoneBoundMark;
    else if (kind == AM_KIND_CRON_SPEC)
      v = repeat_after_from_next(cron_next_utc(c.minute[i], c.hour[i], c.dom[i], c.month[i], c.dow[i], T), T);
    else if (kind == AM_KIND_INTERVAL || kind == AM_KIND_CRON_EVERY)
      v = c.ras[i];
  }
  out[k] = v;
}

// The earliest second after T at which a tick of this shard would emit anything, given the state
// as it is (no further upserts / results): the wake-up time of the reference's earliest timer
// (time.AfterFunc, hcc.go:751) or cron activation (hcc.go:262) — the 1 Hz ticker may sleep until
// then.  Pending results, an unreported "Stopped" and parse errors (requeued after 1 s, hcc.go:204)
// are due at once.  Grid-stride, one record per thread and step; lane -> warp (shuffles) -> global
// atomicMin on a biased unsigned key.  `zone_due`: a lower bound, > T, of the first activation of any
// schedule bound to a named time zone (the launcher derives it from the zones' offsets).  `since`: the hold-in-flight
// column (NULL when the hold is off): a held record is never due by its schedule — its next event is a posted phase
// or a remove, each a reason for the caller to wake the ticker — unless it has a workflow deadline D (`deadline`, NULL
// without workflow timeouts): the tick at max(D, T + 1) times the run out (expire_runs_kernel).
__global__ void next_due_kernel(DevCols c, const int64_t* __restrict__ since, const int64_t* __restrict__ deadline, uint64_t n,
                                int64_t T, int64_t zone_due, unsigned long long* out_biased) {
  unsigned long long best = ~0ull;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t f = c.flags[i];
    const uint32_t kind = f & AM_KIND_MASK;
    if (!is_live(f)) continue;
    int64_t due = INT64_MAX;
    if ((f & kPendBits) || kind == AM_KIND_PARSE_ERROR || (kind == AM_KIND_STOPPED && !(f & AM_F_STOPPED_REPORTED))) {
      due = T + 1;
    } else if (since && held_run(since[i], [&] { return c.finished_at[i]; }, [&] { return f; })) {
      if (deadline && deadline[i] != kNoDeadline) due = deadline[i] > T + 1 ? deadline[i] : T + 1;
    } else if (kind == AM_KIND_INTERVAL || kind == AM_KIND_CRON_EVERY) {
      const int64_t at = (int64_t)((uint64_t)c.finished_at[i] + (uint64_t)(int64_t)c.ras[i]);
      due = ((f & AM_F_TIMER_ARMED) && at > T + 1) ? at : T + 1;
    } else if (kind == AM_KIND_CRON_SPEC && (f >> AM_F_TZ_SHIFT) != 0) {
      due = zone_due;
    } else if (kind == AM_KIND_CRON_SPEC) {
      const int64_t nx = cron_next_utc(c.minute[i], c.hour[i], c.dom[i], c.month[i], c.dow[i], T);
      if (nx != kNoNextFire) due = nx;
    }
    const unsigned long long key = (unsigned long long)due ^ (1ull << 63);  // order-preserving bias
    best = key < best ? key : best;
  }
  best = warp_min(best);
  if ((threadIdx.x & 31) == 0 && best != ~0ull) atomicMin(out_biased, best);
}

// ---- staged controller events (upsert / remove / post_result) ---------------
// Events reach the library from many goroutines between two ticks; per slot
// they must take effect in call order.  An event's tick-local sequence number
// is its position in the staged arrays (1-based).  mark: atomicMax of the sequence into
// the slot's mark triple {latest upsert/remove, latest workflow phase, latest remedy
// phase}; apply: only the marked winners write — the latest upsert/remove, then the latest
// workflow phase and the latest remedy phase if they were posted after it (an older
// result belongs to the replaced CR).  The two phases are tracked independently: the
// reference observes them in separate watch loops (hcc.go:607-756 and :788-852), so a
// "Failed" and a remedy "Succeeded" posted by two calls before one tick must both
// survive.  clear: marks back to zero.  No host-side hashing or sorting.
// A staged op is a uint2 (slot, arg): arg = kind in the top 2 bits; low 30 bits: record index
// (upsert, spec update) or flag bits (result).
// A spec update (am_sweep_update_spec) marks its own word, the slot's latest-spec mark ([cap_padded], allocated at the
// first one): the kernels that take it, and build_planes_dirty_kernel, are instantiated with true for a drain with spec
// updates; a drain without them launches the false instances, which are the kernels of a handle that never stages one.
constexpr uint32_t kOpUpsert = 0u << 30, kOpRemove = 1u << 30, kOpResult = 2u << 30, kOpSpec = 3u << 30;
constexpr uint32_t kOpKindMask = 3u << 30;

// The mark triple of slot i: word x (kMarkState, kMarkHc, kMarkRm) is the 1-based sequence (op k: k + 1) of the slot's
// latest state op (upsert / remove), workflow phase and remedy phase in this drain, 0 for none.  The winner rule below
// works on the words as scalars (held in a struct, they cost the readers registers).
enum : uint32_t { kMarkState = 0u, kMarkHc = 1u, kMarkRm = 2u };
template <typename W>
__device__ __forceinline__ W& mark(W* marks, uint32_t i, uint32_t x) { return marks[3u * i + x]; }
__device__ __forceinline__ bool mark_is(uint32_t word, uint32_t k) { return word == k + 1u; }
__device__ __forceinline__ bool state_op_won(const uint32_t* marks, uint32_t i, uint32_t k) {  // one word read
  return mark(marks, i, kMarkState) == k + 1u;
}
// a phase winner counts when posted after the slot's latest state op (an older result belongs to the replaced CR)
__device__ __forceinline__ bool phase_valid(uint32_t phase, uint32_t state) { return phase != 0u && phase >= state; }
// op k won a phase group: it is the group's winner (`phase`) and that one counts (`valid`)
__device__ __forceinline__ bool phase_won(uint32_t phase, bool valid, uint32_t k) { return valid && mark_is(phase, k); }
// the slot's phases are owned by the workflow-phase winner if it counts, else by the remedy-phase winner
__device__ __forceinline__ bool phase_owner(bool won_hc, bool won_rm, bool hc_valid) {
  return won_hc || (won_rm && !hc_valid);
}
// the posted bits a drain leaves in flags f: each valid winner's arg (fetched only then) replaces its own bit group
template <typename HcArg, typename RmArg>
__device__ __forceinline__ uint32_t merge_phases(uint32_t f, bool hc_valid, HcArg hc_arg, bool rm_valid, RmArg rm_arg) {
  if (hc_valid) f = (f & ~kHcBits) | (hc_arg() & kHcBits);
  if (rm_valid) f = (f & ~kRemedyBits) | (rm_arg() & kRemedyBits);
  return f;
}

template <bool SPEC>
__global__ void mark_ops_kernel(uint32_t* marks, const uint2* __restrict__ ops, uint32_t n, uint32_t* spec_marks) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y;
  if (SPEC && (arg & kOpKindMask) == kOpSpec) { atomicMax(&spec_marks[i], k + 1u); return; }
  if ((arg & kOpKindMask) != kOpResult) { atomicMax(&mark(marks, i, kMarkState), k + 1u); return; }
  if (arg & kHcBits) atomicMax(&mark(marks, i, kMarkHc), k + 1u);
  if (arg & AM_F_REMEDY_PENDING) atomicMax(&mark(marks, i, kMarkRm), k + 1u);
}

// upserts (hcc.go:170-188 Reconcile) and removes (hcc.go:175-186).  Both may change the slot's kind or
// masks: its segment is marked for build_planes_dirty_kernel.
__global__ void apply_state_ops_kernel(DevCols c, const uint32_t* __restrict__ marks, const uint2* __restrict__ ops,
                                       const am_record_t* __restrict__ recs, uint32_t n, uint32_t* seg_dirty,
                                       uint32_t* due, int64_t due_epoch) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y;
  const uint32_t kind = arg & kOpKindMask;
  if (kind == kOpResult || !state_op_won(marks, i, k)) return;
  seg_dirty[i / kRecPerWarp] = 1u;
  if (kind == kOpRemove) { c.flags[i] = AM_F_TOMBSTONE; return; }
  const am_record_t r = recs[arg & ~kOpKindMask];
  c.minute[i] = r.minute; c.hour[i] = r.hour; c.dom[i] = r.dom; c.month[i] = r.month; c.dow[i] = r.dow;
  c.ras[i] = r.ras; c.flags[i] = r.flags; c.finished_at[i] = r.finished_at;
  c.runs_limit[i] = r.runs_limit; c.reset_interval[i] = r.reset_interval;
  c.success[i] = r.success; c.failed[i] = r.failed; c.remedy_success[i] = r.remedy_success;
  c.remedy_failed[i] = r.remedy_failed; c.remedy_total[i] = r.remedy_total;
  c.remedy_finished_at[i] = r.remedy_finished_at;
  if (due) due[i] = due_word(r.ras, r.finished_at, due_epoch);
}

// ---- the mask bit planes (MaskPlanes) --------------------------------------
// bit v of a record's masks for plane P (the star plane: bit 63 of dom or dow)
__device__ __forceinline__ bool plane_bit(int P, uint64_t mi, uint64_t hr, uint64_t dm, uint64_t mo, uint64_t dw) {
  if (P < kPlaneHour) return (mi >> (P - kPlaneMinute)) & 1u;
  if (P <= kPlaneDom) return (hr >> (P - kPlaneHour)) & 1u;
  if (P <= kPlaneMonth) return (dm >> (P - kPlaneDom)) & 1u;
  if (P < kPlaneDow) return (mo >> (P - kPlaneMonth)) & 1u;
  if (P < kPlaneStar) return (dw >> (P - kPlaneDow)) & 1u;
  return ((dm | dw) >> 63) != 0;
}

// Rebuild the plane words of segment `seg` with one warp, a 32-record quarter (one word per plane) at a
// time: lane L reads record 32q + L of the segment, one ballot per plane gives the word, and lane L
// stores planes L, L + 32, ...
__device__ __forceinline__ void build_segment_planes(const DevCols& c, const MaskPlanes& pl, uint32_t seg, int lane) {
  for (uint32_t q = 0; q < (uint32_t)kRecPerWarp / 32u; ++q) {
    const uint32_t wq = seg * (uint32_t)(kRecPerWarp / 32) + q;
    const uint32_t i = wq * 32u + (uint32_t)lane;
    const uint32_t f = c.flags[i];
    const bool on = (f & AM_KIND_MASK) == AM_KIND_CRON_SPEC && (f >> AM_F_TZ_SHIFT) == 0;
    const uint64_t mi = c.minute[i], hr = c.hour[i], dm = c.dom[i], mo = c.month[i], dw = c.dow[i];
    uint32_t mine[(kPlanes + 31) / 32] = {};
#pragma unroll
    for (int P = 0; P < kPlanes; ++P) {
      const uint32_t b = __ballot_sync(kFull, on && plane_bit(P, mi, hr, dm, mo, dw));
      if ((P & 31) == lane) mine[P / 32] = b;
    }
#pragma unroll
    for (int k = 0; k < (kPlanes + 31) / 32; ++k) {
      const uint32_t P = (uint32_t)(32 * k + lane);
      if (P < (uint32_t)kPlanes) pl.w[P * pl.words + wq] = mine[k];
    }
  }
}
static_assert(kRecPerWarp % 32 == 0, "build_segment_planes: whole plane words per segment");

// every segment of [seg0, seg0 + n_seg), one warp each (am_sweep_load_range)
__global__ void build_planes_range_kernel(DevCols c, MaskPlanes pl, uint32_t seg0, uint32_t n_seg) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n_seg) return;  // warp-uniform
  build_segment_planes(c, pl, seg0 + w, (int)(threadIdx.x & 31));
}

// After apply_state_ops_kernel: one warp per staged op.  The first warp that claims a segment marked
// there rebuilds it, so the cost is one claim per op plus one rebuild per segment touched.  PEEK (drains with spec
// updates, which mark only the segments whose masks, kinds or zones changed): the claim is tried only where a plain
// load finds the mark, so the ops of clean segments, up to 128 per segment, do not queue on its word's atomic.
template <bool PEEK>
__global__ void build_planes_dirty_kernel(DevCols c, MaskPlanes pl, uint32_t* seg_dirty, const uint2* __restrict__ ops,
                                          uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (k >= n) return;  // warp-uniform
  const int lane = (int)(threadIdx.x & 31);
  const uint32_t seg = ops[k].x / (uint32_t)kRecPerWarp;
  const bool won =
      lane == 0 && (!PEEK || seg_dirty[seg] != 0u) && atomicAnd(&seg_dirty[seg], 0u) != 0u;  // (an exchange with 0)
  if (__ballot_sync(kFull, won)) build_segment_planes(c, pl, seg, lane);
}

// terminal phases observed by the watch loops (hcc.go:635/:662/:821/:836).  The winner of
// the workflow phase and the winner of the remedy phase may be two different ops of the
// same slot: each rewrites only its own bit group, atomically.
__global__ void apply_result_ops_kernel(uint32_t* flags, const uint32_t* __restrict__ marks, const uint2* __restrict__ ops,
                                        uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y;
  if ((arg & kOpKindMask) != kOpResult) return;
  // the winner rule with one word read per test, spelled as compares (through mark_is the kernel compiles differently)
  if (k + 1u < mark(marks, i, kMarkState)) return;
  uint32_t clr = 0, set = 0;
  if ((arg & kHcBits) && mark(marks, i, kMarkHc) == k + 1u) { clr |= kHcBits; set |= arg & kHcBits; }
  if ((arg & AM_F_REMEDY_PENDING) && mark(marks, i, kMarkRm) == k + 1u) { clr |= kRemedyBits; set |= arg & kRemedyBits; }
  if (clr) {
    atomicAnd(&flags[i], ~clr);
    atomicOr(&flags[i], set);
  }
}

// Results posted between two ticks, applied while the tick drains them instead of inside its sweep.
// In the sweep a record with a posted result costs its warp a second, dependent memory round trip
// (the remedy / counter columns) behind the streaming loads; with a result on ~2 % of the records
// nine warps in ten pay it and the tick's sweep slows markedly at 10 M records.
// Here every result is its own thread: the slot's owner (see below)
// merges the posted bits into the flags, gathers the state columns its case needs, runs the same
// apply_result and scatters what changed — this kernel REPLACES apply_result_ops_kernel for such a drain.  The action bits go
// into the flags' carry bits for the sweep of the SAME tick to emit (it clears them); the finishedAt /
// timer-armed state it leaves is exactly what the sweep's own step 1 would have decided on.  Only the
// tick's drain does this (T is the tick's second) and only when results are sparse; a read drains
// without it, and a dense batch is cheaper as the sweep's streaming path.
// REMEDY (remedy hold): a result that runs the remedy without a remedy outcome merged starts a remedy run here
// (start_remedy_run; `deadline` NULL without timeout state), and the sweep of the same tick holds the record.
template <bool REMEDY>
__global__ void apply_results_now_kernel(DevCols c, const uint32_t* __restrict__ marks, const uint2* __restrict__ ops, uint32_t n,
                                         int64_t T, unsigned long long* acc, int64_t* since, int64_t* deadline,
                                         const int32_t* __restrict__ wf_timeout, unsigned long long* seg_deadline,
                                         uint32_t* due, int64_t due_epoch) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t res = 0;
  uint2 op = make_uint2(0u, 0u);
  if (k < n) op = ops[k];
  if (k < n && (op.y & kOpKindMask) == kOpResult) {
    const uint32_t i = op.x, arg = op.y;
    const uint32_t s_state = mark(marks, i, kMarkState), hcw = mark(marks, i, kMarkHc), rmw = mark(marks, i, kMarkRm);
    const bool hc_valid = phase_valid(hcw, s_state), rm_valid = phase_valid(rmw, s_state);
    // The winners of the slot's two phase groups may be two different ops; ONE thread owns the slot here
    // (phase_owner) and takes the other group's bits from that op, so the flags are read and written once, without
    // atomics.  The owner is the workflow-phase winner whenever that one is valid.
    const bool won_hc = phase_won(hcw, hc_valid, k), won_rm = phase_won(rmw, rm_valid, k);
    if (phase_owner(won_hc, won_rm, hc_valid)) {  // (so a valid workflow winner is this op: won_hc == hc_valid)
      const uint32_t f = merge_phases(c.flags[i], won_hc, [&] { return arg; }, rm_valid,
                                      [&] { return won_rm ? arg : ops[rmw - 1u].y; });
      if (!is_live(f) || !(f & kPendBits)) {
        c.flags[i] = f;  // (a record the sweep does not evaluate keeps its posted result)
      } else {
        // Gather only what this result can touch (every column is its own 32-B sector of a random record):
        // a "Succeeded" on a check without remedy reads its success counter and nothing else — two gathers
        // instead of ten; with all ten the kernel took as long as the sweep's own
        // sparse path it replaces.  What apply_result reads, by case (hcc.go:635-724, :821-851):
        //   Succeeded: SuccessCount;            with a remedy workflow: RemedyTotalRuns (reset on pass)
        //   Failed:    FailedCount;             with a remedy workflow: the gate (limit, reset interval, total, finishedAt)
        //   a remedy outcome (applied only behind a Failed that runs the remedy, or on its own): the remedy counters
        const bool r_ok = (f & AM_F_PENDING_OK) != 0, r_fail = !r_ok && (f & AM_F_PENDING_FAIL) != 0;
        const bool remedy_state = ((r_ok || r_fail) && (f & AM_F_HAS_REMEDY)) || (!r_ok && !r_fail);
        RecState s{};
        s.flags = f;  // (finishedAt is only ever overwritten with T by a workflow result: not read)
        if (r_ok) s.s = c.success[i];
        if (r_fail) s.f = c.failed[i];
        if (remedy_state) {
          s.rs = c.remedy_success[i]; s.rf = c.remedy_failed[i]; s.rt = c.remedy_total[i];
          s.rfa = c.remedy_finished_at[i]; s.limit = c.runs_limit[i]; s.reset = c.reset_interval[i];
        }
        const RecState b = s;
        const uint32_t a = apply_result(s, T, res);
        if (r_ok || r_fail) {
          c.finished_at[i] = s.fa;
          if (due) due[i] = due_word(c.ras[i], s.fa, due_epoch);
        }
        if (s.s != b.s) c.success[i] = s.s;
        if (s.f != b.f) c.failed[i] = s.f;
        if (s.rs != b.rs) c.remedy_success[i] = s.rs;
        if (s.rf != b.rf) c.remedy_failed[i] = s.rf;
        if (s.rt != b.rt) c.remedy_total[i] = s.rt;
        if (s.rfa != b.rfa) c.remedy_finished_at[i] = s.rfa;
        c.flags[i] = s.flags | carry_of_actions(a);  // pending bits cleared, timer armed, action bits for this tick's sweep
        if (REMEDY && starts_remedy_run(a, f)) {
          if (deadline) start_remedy_run<true>(since, deadline, wf_timeout, seg_deadline, i, T);
          else start_remedy_run<false>(since, deadline, wf_timeout, seg_deadline, i, T);
        }
      }
    }
  }
  // results applied (metrics.MonitorSuccess / Error): warp -> global RED, as the sweep does per tile
  const int lane = threadIdx.x & 31;
  const uint32_t v = warp_result_count(res, lane);
  if (lane < 4 && v) atomicAdd(&acc[10 + lane], (unsigned long long)v);
}

// Hold in flight: the drain's staged ops that end a run clear the slot's since.
//   * a workflow phase (Succeeded / Failed): the run is over (hcc.go:635/:662), whatever else the drain does — also
//     when a later upsert of the slot supersedes the result itself, and whatever second the next tick has;
//   * a remove: no workflow in flight any more (hcc.go:175-186 stops its timer), also one followed by an upsert of the
//     same slot (a new CR in an old slot).
// A remedy phase alone ends a remedy run (remedy hold: hcc.go:821-851 end watchRemedyWorkflow), not a health-check run.
// Launched only while the hold is on.
__global__ void clear_since_kernel(int64_t* since, const uint2* __restrict__ ops, uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: the previous tick's sweep writes since)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t kind = op.y & kOpKindMask;
  if (kind == kOpRemove || (kind == kOpResult && (op.y & kHcBits))) since[op.x] = kNotInFlight;
  else if (kind == kOpResult && (op.y & AM_F_REMEDY_PENDING) && is_remedy_run(since[op.x])) since[op.x] = kNotInFlight;
}

// Turning the remedy hold off: every remedy run ends, with its deadline (`deadline` NULL without timeout state).
__global__ void release_remedy_runs_kernel(int64_t* since, int64_t* deadline, uint64_t n) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (is_remedy_run(since[i])) {
      since[i] = kNotInFlight;
      if (deadline) deadline[i] = kNoDeadline;
    }
  }
}

__global__ void fill_i64_kernel(int64_t* p, int64_t v, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// What am_sweep_in_flight reports for slot i: since of a slot the next tick would hold (the sweep's rule, on the drained
// state) for a health-check run, else kNotInFlight.  `remedy` (am_sweep_remedy_in_flight): the start of a held remedy
// run instead.  finishedAt and the flags are read only for a slot whose since is set.  The one definition of both
// values: the dense queries and am_sweep_select's mark pass call it.
__device__ __forceinline__ int64_t held_run_start(const DevCols& c, const int64_t* __restrict__ since, uint32_t i,
                                                  bool remedy) {
  const int64_t s = since[i];
  const bool held = held_run(s, [&] { return c.finished_at[i]; }, [&] { return c.flags[i]; });
  return held && is_remedy_run(s) == remedy ? run_start(s) : kNotInFlight;
}

// am_sweep_in_flight / am_sweep_remedy_in_flight: held_run_start of the slots first + k (idx == NULL) or first + idx[k],
// k < n.
__global__ void in_flight_kernel(DevCols c, const int64_t* __restrict__ since, uint32_t first, const uint32_t* __restrict__ idx,
                                 uint32_t n, int64_t* out, bool remedy) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  out[k] = held_run_start(c, since, first + (idx ? idx[k] : k), remedy);
}

// Workflow timeouts: the drain's winning upserts (the marks decide, as in apply_state_ops_kernel) store their record's
// wf_timeout.  The timeout of a run is read when the sweep submits it, so an upsert during a run changes the next run's.
// Launched with every drain that has state ops once the handle has timeout state.
__global__ void store_wf_timeout_kernel(int32_t* wf, const uint32_t* __restrict__ marks, const uint2* __restrict__ ops,
                                        const am_record_t* __restrict__ recs, uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y;
  if ((arg & kOpKindMask) != kOpUpsert || !state_op_won(marks, i, k)) return;
  wf[i] = recs[arg & ~kOpKindMask].wf_timeout;
}

// Workflow timeouts at a tick (hcc.go:613 NewIEBWithTimeout with Spec.Workflow.Timeout; :627-632 the watch loop posts a
// synthetic "Failed" when the run outlives it).  Runs in the tick's drain while the hold is on, after clear_since_kernel
// and before the result kernels.  Lane L of a warp reads the bound of segment 32 w + L: 8 B per 128 slots when nothing
// is due.  A segment whose bound is <= T is visited by the whole warp, 32 slots at a time: every deadline <= T is
// dropped; a run that is still held (the sweep's rule) on a live record gets AM_F_PENDING_FAIL, exactly as a posted
// Failed does, so the result kernel behind this one or the sweep's pending path applies it (counters, finishedAt = T,
// timer, remedy gate); its since is cleared as clear_since_kernel clears it for a posted phase; and (slot, since) is
// appended to the tick's list (one atomic per segment).  The bound becomes the exact minimum of what is left.  A remedy
// run (remedy hold) gets AM_F_REMEDY_PENDING without the OK bit instead, and its since word goes into the list as it
// is: the host tells the two kinds apart.
__global__ void expire_runs_kernel(DevCols c, int64_t* since, int64_t* deadline, unsigned long long* seg_deadline,
                                   uint32_t n_seg, int64_t T, uint32_t* out_idx, int64_t* out_since, uint32_t* out_count) {
  pdl_wait();  // (launched with programmatic stream serialisation: the previous tick's sweep writes deadlines)
  const int lane = threadIdx.x & 31;
  const uint32_t seg0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32u;
  if (seg0 >= n_seg) return;  // warp-uniform
  const unsigned long long tkey = biased_key(T);
  uint32_t due = __ballot_sync(kFull, seg0 + (uint32_t)lane < n_seg && seg_deadline[seg0 + lane] <= tkey);
  while (due) {  // warp-uniform
    const uint32_t seg = seg0 + (uint32_t)(__ffs((int)due) - 1);
    due &= due - 1;
    unsigned long long left = ~0ull;
    uint32_t hit = 0;  // bit q: slot 32 q + lane of the segment timed out
    int64_t sv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t i = seg * (uint32_t)kRecPerWarp + 32u * q + (uint32_t)lane;
      const int64_t D = deadline[i];
      sv[q] = kNotInFlight;
      if (D <= T) {
        deadline[i] = kNoDeadline;
        const uint32_t f = c.flags[i];
        const int64_t s = since[i];
        // held_run, written out: through the call this kernel compiles to different machine code
        if (is_live(f) && s != kNotInFlight && s >= c.finished_at[i] && !(f & kHcBits)) {
          // a remedy run (remedy hold, hcc.go:813-818) times out as a posted remedy "Failed"
          c.flags[i] = is_remedy_run(s) ? ((f & ~AM_F_REMEDY_OUTCOME_OK) | AM_F_REMEDY_PENDING) : (f | AM_F_PENDING_FAIL);
          since[i] = kNotInFlight;
          sv[q] = s;
          hit |= 1u << q;
        }
      } else if (biased_key(D) < left) {
        left = biased_key(D);
      }
    }
    const uint32_t cnt = (uint32_t)__popc(hit);
    const uint32_t incl = warp_inclusive_scan(cnt, lane);
    const uint32_t total = __reduce_add_sync(kFull, cnt);
    uint32_t base = 0;
    if (total && lane == 0) base = atomicAdd(out_count, total);
    base = __reduce_add_sync(kFull, base);  // (lane 0's, to every lane)
    uint32_t pos = base + incl - cnt;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if ((hit >> q) & 1u) {
        out_idx[pos] = seg * (uint32_t)kRecPerWarp + 32u * q + (uint32_t)lane;
        out_since[pos] = sv[q];
        ++pos;
      }
    }
    left = warp_min(left);
    if (lane == 0) seg_deadline[seg] = left;
  }
}

// ---- simulated workflows (am_sweep_simulate) ----------------------------------------------------------------------
// The durations of the two kinds of run: min and max - min + 1, in seconds.
struct SimDraw {
  uint64_t seed;
  int32_t wf_min, wf_span, remedy_min, remedy_span;
};

// The simulated end of the run a since word holds (either kind), and the phase bits its end posts (*bits: a workflow
// phase for a health-check run, a remedy phase for a remedy run).  A pure function of the run's start: the keyed
// splitmix64 of the closed loop (outcome_key) decides both, the outcome from its low bytes as the closed loop does
// (the record's fail_p8 for a health check, 179/256 for a remedy), the duration from its high word.
__device__ __forceinline__ int64_t sim_run_end(const SimDraw& q, uint64_t g, int64_t since, uint32_t flags, uint32_t* bits) {
  const bool remedy = is_remedy_run(since);
  const int64_t start = run_start(since);
  const uint64_t k = outcome_key(q.seed, g, (uint64_t)start);
  if (remedy) {
    *bits = AM_F_REMEDY_PENDING | ((uint32_t)((k >> 8) & 0xFF) < 179u ? AM_F_REMEDY_OUTCOME_OK : 0u);
    return start + q.remedy_min + (int64_t)((k >> 32) % (uint64_t)q.remedy_span);
  }
  *bits = (uint32_t)(k & 0xFF) < ((flags >> AM_F_FAILP_SHIFT) & 0xFFu) ? AM_F_PENDING_FAIL : AM_F_PENDING_OK;
  return start + q.wf_min + (int64_t)((k >> 32) % (uint64_t)q.wf_span);
}

// The simulated post of a run that ends: its phase replaces its bit group, as am_sweep_post_result stages it.
__device__ __forceinline__ uint32_t sim_post(uint32_t f, uint32_t bits) {
  return (f & ~((bits & kHcBits) ? kHcBits : kRemedyBits)) | bits;
}

// The completion pass of a simulated tick at T, ahead of its expiry pass: every held run (held_run, either kind) whose
// simulated end is <= T posts its phase into the flags and clears since, as the drain of a posted phase does
// (apply_result_ops_kernel, clear_since_kernel).  Shaped like expire_runs_kernel: lane L of a warp reads the bound of
// segment 32 w + L (`seg_end`, a lower bound of the segment's simulated ends); a segment whose bound is <= T is visited
// by the whole warp and gets the exact minimum of what is left.  A segment's bound is lowered when a tick starts a run
// in it (sim_note_starts_kernel).
__global__ void sim_complete_kernel(DevCols c, int64_t* since, unsigned long long* seg_end, uint32_t n_seg, int64_t T,
                                    SimDraw q, uint64_t shard_base) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const uint32_t seg0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32u;
  if (seg0 >= n_seg) return;  // warp-uniform
  const unsigned long long tkey = biased_key(T);
  uint32_t due = __ballot_sync(kFull, seg0 + (uint32_t)lane < n_seg && seg_end[seg0 + lane] <= tkey);
  while (due) {  // warp-uniform
    const uint32_t seg = seg0 + (uint32_t)(__ffs((int)due) - 1);
    due &= due - 1;
    unsigned long long left = ~0ull;
#pragma unroll
    for (int q4 = 0; q4 < 4; ++q4) {
      const uint32_t i = seg * (uint32_t)kRecPerWarp + 32u * q4 + (uint32_t)lane;
      const int64_t s = since[i];
      if (s == kNotInFlight) continue;
      const uint32_t f = c.flags[i];
      if (!held_run(s, [&] { return c.finished_at[i]; }, [&] { return f; })) continue;
      uint32_t bits;
      const int64_t end = sim_run_end(q, shard_base + i, s, f, &bits);
      if (end <= T) {
        c.flags[i] = sim_post(f, bits);
        since[i] = kNotInFlight;
      } else if (biased_key(end) < left) {
        left = biased_key(end);
      }
    }
    left = warp_min(left);
    if (lane == 0) seg_end[seg] = left;
  }
}

// The bounds of sim_complete_kernel from the since words as they stand: every held run's simulated end, per segment
// (`seg_end` all ones on entry).  One thread per slot; a warp's 32 slots lie in one segment.
__global__ void sim_bounds_kernel(DevCols c, const int64_t* __restrict__ since, unsigned long long* seg_end, uint64_t n,
                                  SimDraw q, uint64_t shard_base) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned long long key = ~0ull;
  if (i < n) {
    const int64_t s = since[i];
    if (s != kNotInFlight) {
      const uint32_t f = c.flags[i];
      uint32_t bits;
      if (held_run(s, [&] { return c.finished_at[i]; }, [&] { return f; }))
        key = biased_key(sim_run_end(q, shard_base + i, s, f, &bits));
    }
  }
  key = warp_min(key);
  if ((threadIdx.x & 31) == 0 && key != ~0ull) atomicMin(seg_end + i / (uint64_t)kRecPerWarp, key);
}

// After a simulated tick's sweep: every run it started is a record it emitted (SUBMIT_HC, or RUN_REMEDY for a remedy
// run), and no run ends before T + the shorter minimum duration (`earliest`).  So a segment with an emitted record in
// the tick's bitmap gets its bound lowered to that.  One thread per segment (four bitmap words).
__global__ void sim_note_starts_kernel(const uint32_t* __restrict__ bitmap, unsigned long long* seg_end, uint32_t n_seg,
                                       int64_t earliest) {
  pdl_wait();
  const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
  if (seg >= n_seg) return;
  const uint4 w = *reinterpret_cast<const uint4*>(bitmap + 4ull * seg);
  if ((w.x | w.y | w.z | w.w) && biased_key(earliest) < seg_end[seg]) seg_end[seg] = biased_key(earliest);
}

// The counts of a simulated tick's row (am_sim_tick_t, zero on entry) after its sweep: the held runs of either kind, as
// am_sweep_in_flight / am_sweep_remedy_in_flight report them, and the tick's timed-out list split by kind (`to_count`
// NULL when the tick ran no expiry pass).  Grid-stride.
__global__ void sim_count_kernel(DevCols c, const int64_t* __restrict__ since, uint64_t n, const int64_t* __restrict__ to_since,
                                 const uint32_t* __restrict__ to_count, unsigned long long* row) {
  pdl_wait();
  uint32_t hc = 0, rm = 0, to = 0, rto = 0;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t s = since[i];
    if (s != kNotInFlight && held_run(s, [&] { return c.finished_at[i]; }, [&] { return c.flags[i]; })) {
      if (is_remedy_run(s)) ++rm; else ++hc;
    }
  }
  const uint32_t m = to_count ? *to_count : 0u;
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < m; k += stride) {
    if (is_remedy_run(to_since[k])) ++rto; else ++to;
  }
  const uint32_t v[4] = {hc, rm, to, rto};
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    const uint32_t t = __reduce_add_sync(kFull, v[f]);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(row + f, (unsigned long long)t);
  }
}

template <bool SPEC>
__global__ void clear_marks_kernel(uint32_t* marks, const uint2* __restrict__ ops, uint32_t n, uint32_t* spec_marks) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = ops[k].x;
#pragma unroll
  for (uint32_t x = kMarkState; x <= kMarkRm; ++x) mark(marks, i, x) = 0;
  if (SPEC) spec_marks[i] = 0;
}

// ---- status changes (am_sweep_set_track_changes) --------------------------------------------------------------
// The handle keeps one bit per slot, bit i & 31 of word i / 32: "the coming tick changes this slot's columns".  Drains
// add to it (a read's drain too: the results it leaves pending belong to the next tick), the tick adds and removes what
// only the sweep decides, and after the sweep the bits are compacted into the tick's ascending slot list and cleared.
// A set bit whose slot is not live when the list is built is dropped: the result kernels and the sweep apply nothing to
// such a slot, and nothing between the drain and the list changes a kind or a tombstone.

// A drain's staged ops, after apply_state_ops_kernel and before anything applies a result.  One thread per slot decides
// (the marks' rules, as in apply_results_now_kernel): the slot's latest upsert / remove, else its workflow-phase winner,
// else its remedy-phase winner.  With an upsert or remove the bit is set exactly when a phase posted after it survives
// or the upserted record itself carries pending results; an older bit (a read's drain left a result pending) goes, as
// the state op overwrote that result.  Without one, a surviving phase sets the bit.
__global__ void note_ops_kernel(uint32_t* bits, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ marks,
                                const uint2* __restrict__ ops, uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = ops[k].x;
  const uint32_t s_state = mark(marks, i, kMarkState), hcw = mark(marks, i, kMarkHc), rmw = mark(marks, i, kMarkRm);
  const bool hc_valid = phase_valid(hcw, s_state), rm_valid = phase_valid(rmw, s_state);
  uint32_t* w = bits + i / 32u;
  const uint32_t b = 1u << (i & 31u);
  if (s_state) {
    if (!mark_is(s_state, k)) return;
    if (hc_valid || rm_valid || (flags[i] & kPendBits)) atomicOr(w, b);
    else atomicAnd(w, ~b);
  } else if (phase_owner(phase_won(hcw, hc_valid, k), phase_won(rmw, rm_valid, k), hc_valid)) {
    atomicOr(w, b);
  }
}

// The slots of a device list of *count entries (the expiry pass's timed-out runs, each given a pending Failed): set.
// Grid-stride: the count is known on the device only.
__global__ void note_slots_kernel(uint32_t* bits, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ count) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t n = *count;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    atomicOr(bits + idx[k] / 32u, 1u << (idx[k] & 31u));
}

// The bits of slots [first, first + n) from their flags alone: set where a live record carries a pending result.  Turning
// tracking on (every slot) and am_sweep_load_range (its range) start from here.  One thread per word; the partial words
// at either end keep their other bits.
__global__ void seed_changes_kernel(uint32_t* bits, const uint32_t* __restrict__ flags, uint64_t first, uint64_t n) {
  const uint64_t w0 = first / 32u, w1 = (first + n + 31u) / 32u;
  for (uint64_t w = w0 + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < w1; w += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t in = 0, v = 0;
    for (uint32_t b = 0; b < 32u; ++b) {
      const uint64_t i = w * 32u + b;
      if (i < first || i >= first + n) continue;
      in |= 1u << b;
      const uint32_t f = flags[i];
      if (is_live(f) && (f & kPendBits)) v |= 1u << b;
    }
    if (in == kFull) {
      bits[w] = v;
    } else {
      atomicAnd(bits + w, ~in);
      atomicOr(bits + w, v);
    }
  }
}

// After the sweep, one warp per tile, over the tile's exceptions (the non-default actions it emitted): a record reported
// STOPPED is in (finishedAt = T and STOPPED_REPORTED); otherwise one whose result came out AM_ACT_ANOMALY is out (the
// reference panics at hcc.go:690 before it writes a status, DESIGN.md section 6 item 5).  `closed` (closed loop): every
// record emitted with SUBMIT_HC completed in this tick, so the tile's emitted bits are OR-ed in first (lane L: word L),
// and an exception without SUBMIT_HC keeps the bit it had before (a result, if any, set it at the drain).
__global__ void note_exceptions_kernel(uint32_t* bits, const TickOut out, uint32_t n_tiles, bool closed) {
  __shared__ uint32_t s_before[kWarps][kTileWords];
  pdl_wait();  // (launched with programmatic stream serialisation: the sweep writes the exceptions)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t tile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (tile >= n_tiles) return;  // warp-uniform
  uint32_t* w = bits + (size_t)tile * kTileWords;
  if (closed) {
    const uint32_t before = w[lane];
    s_before[warp][lane] = before;
    w[lane] = before | out.bitmap[(size_t)tile * kTileWords + lane];
  }
  __syncwarp();
  const uint32_t ne = out.tile_exc[tile];
  for (uint32_t e = (uint32_t)lane; e < ne; e += 32u) {
    const uint32_t x = out.exc_seg[(size_t)tile * kTile + e];
    const uint32_t off = exc_offset(x), a = exc_action(x), b = 1u << (off & 31u);
    if (a & AM_ACT_STOPPED) atomicOr(w + off / 32u, b);
    else if ((a & AM_ACT_ANOMALY) || (closed && !(a & AM_ACT_SUBMIT_HC) && !(s_before[warp][off / 32u] & b)))
      atomicAnd(w + off / 32u, ~b);
  }
}

// The list, in two passes of one CTA per 8192-slot group (thread t: word t of the group) around scan_groups_kernel.
// Counting drops the bits of slots that are not live; listing writes the group's slots at its offset, ascending, and
// clears the words.  Groups with nothing listed are not read twice.
__global__ void __launch_bounds__(kGroupWords) count_changes_kernel(uint32_t* bits, const uint32_t* __restrict__ flags,
                                                                    uint32_t* group_count) {
  __shared__ uint32_t s_warp[kGroupWords / 32];
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t wi = (size_t)blockIdx.x * kGroupWords + threadIdx.x;
  uint32_t v = bits[wi];
  if (v) {
    uint32_t keep = v;
    for (uint32_t m = v; m; m &= m - 1u) {
      const uint32_t b = (uint32_t)__ffs((int)m) - 1u;
      if (!is_live(flags[wi * 32u + b])) keep &= ~(1u << b);
    }
    if (keep != v) bits[wi] = keep;
    v = keep;
  }
  const uint32_t c = __reduce_add_sync(kFull, (uint32_t)__popc(v));
  if (lane == 0) s_warp[warp] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (uint32_t k = 0; k < kGroupWords / 32u; ++k) t += s_warp[k];
    group_count[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kGroupWords) list_changes_kernel(uint32_t* bits, const uint32_t* __restrict__ group_prefix,
                                                                   uint32_t* list) {
  __shared__ uint32_t s_warp[kGroupWords / 32];
  pdl_wait();  // (launched with programmatic stream serialisation: scan_groups_kernel writes the offsets)
  const uint32_t g = blockIdx.x;
  const uint32_t base = group_prefix[g];
  if (group_prefix[g + 1u] == base) return;  // block-uniform
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t wi = (size_t)g * kGroupWords + threadIdx.x;
  const uint32_t v = bits[wi];
  const uint32_t c = (uint32_t)__popc(v);
  const uint32_t incl = warp_inclusive_scan(c, lane);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t pos = base + incl - c;
  for (int k = 0; k < warp; ++k) pos += s_warp[k];
  for (uint32_t m = v; m; m &= m - 1u) list[pos++] = (uint32_t)(wi * 32u) + (uint32_t)__ffs((int)m) - 1u;
  if (v) bits[wi] = 0;
}

// ---- change details (am_sweep_set_change_details) -------------------------------------------------------------
// Per slot, beside the status-change bit: `applied`, the AM_CHG_* bits of the results the coming tick applies, and
// `start`, the start of the run whose phase it applies as a since word (T, or T + kRemedyRun for a remedy run;
// kNotInFlight when none).  A slot has at most one run in flight, so one word serves both kinds.  The pair is
// meaningful exactly while the slot's status-change bit is set: every pass that sets the bit writes the pair first,
// and a pass that finds the bit clear starts from (0, kNotInFlight).  Nothing clears them after a tick: the tick
// copies the pairs of its list, by entry, into a second pair of arrays (snapshot_details_kernel).
// A result op carries its post call's tag in arg bits 8..29 (am_sweep_post_result: the call's first op index, mod
// 2^22), which no other kernel reads: two entries of one call see the same in-flight state, as they do in call order.
// Within a drain of at most kCallTagSpan ops equal tags mean one call; a longer drain also hands the kernel the first
// op index of every post call.
constexpr uint32_t kCallTagShift = 8, kCallTagSpan = 1u << 22, kCallTagMask = (kCallTagSpan - 1u) << kCallTagShift;
static_assert((kCallTagMask & (kOpKindMask | kHcBits | kRemedyBits)) == 0, "call tag bits");

// The AM_CHG_* bits of a flags word's posted-result bits.
__device__ __forceinline__ uint32_t applied_of(uint32_t f) {
  return ((f & AM_F_PENDING_OK) ? AM_CHG_SUCCEEDED : 0u) | ((f & AM_F_PENDING_FAIL) ? AM_CHG_FAILED : 0u) |
         ((f & AM_F_REMEDY_PENDING) ? ((f & AM_F_REMEDY_OUTCOME_OK) ? AM_CHG_REMEDY_SUCCEEDED : AM_CHG_REMEDY_FAILED) : 0u);
}

// A drain's ops, after apply_state_ops_kernel and before clear_since_kernel and the result kernels (the flags hold the
// already-pending bits, since the in-flight state before the drain).  The slot's owner (note_ops_kernel's: its latest
// upsert / remove, else its workflow-phase winner, else its remedy-phase winner) writes the pair: applied from the
// posted bits the drain leaves (merge_phases, the result kernels' rule); start from the held run (held_run) when
// a winner of its kind ends it, else an earlier drain's capture whose phase is still pending and not replaced.  A
// state op drops the earlier capture (the record's own pending bits report no start).  `since` NULL: the hold is off.
// capture_superseded_kernel then drops a capture that an earlier call of the drain ended first.
__global__ void capture_ops_kernel(uint8_t* applied, int64_t* start, const DevCols c, const int64_t* __restrict__ since,
                                   const uint32_t* __restrict__ marks, const uint2* __restrict__ ops, uint32_t n) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = ops[k].x;
  const uint32_t s_state = mark(marks, i, kMarkState), hcw = mark(marks, i, kMarkHc), rmw = mark(marks, i, kMarkRm);
  const bool hc_valid = phase_valid(hcw, s_state), rm_valid = phase_valid(rmw, s_state);
  if (s_state ? !mark_is(s_state, k) : !phase_owner(phase_won(hcw, hc_valid, k), phase_won(rmw, rm_valid, k), hc_valid))
    return;
  const uint32_t f = c.flags[i];
  const uint32_t fm = merge_phases(f, hc_valid, [&] { return ops[hcw - 1u].y; }, rm_valid, [&] { return ops[rmw - 1u].y; });
  int64_t w = kNotInFlight;
  if (!s_state) {
    const int64_t old = start[i];
    const bool rem = is_remedy_run(old);
    if (old != kNotInFlight && !(rem ? rm_valid : hc_valid) && (f & (rem ? AM_F_REMEDY_PENDING : kHcBits))) w = old;
  }
  if (since) {
    const int64_t s = since[i];
    if (held_run(s, [&] { return c.finished_at[i]; }, [&] { return f; }) && (is_remedy_run(s) ? rm_valid : hc_valid))
      w = s;
  }
  start[i] = w;
  applied[i] = (uint8_t)applied_of(fm);
}

// After capture_ops_kernel, one thread per op: an op that ended the captured run before the winner's call did (a
// remove; a workflow phase; for a remedy run any phase) leaves the winner's call nothing in flight.  A spec update ends
// nothing.  `calls` (NULL when the drain has at most kCallTagSpan ops): the n_calls first op indices of the drain's post
// calls, ascending; two result ops with equal tags are of one call iff no call starts after the first, up to the second.
template <bool SPEC>
__global__ void capture_superseded_kernel(int64_t* start, const uint32_t* __restrict__ marks, const uint2* __restrict__ ops,
                                          uint32_t n, const uint32_t* __restrict__ calls, uint32_t n_calls) {
  pdl_wait();  // (launched with programmatic stream serialisation: capture_ops_kernel writes start)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y, kind = arg & kOpKindMask;
  if (kind == kOpUpsert || (SPEC && kind == kOpSpec)) return;
  const int64_t w = start[i];
  if (w == kNotInFlight) return;
  const bool rem = is_remedy_run(w);
  const uint32_t win = mark(marks, i, rem ? kMarkRm : kMarkHc);
  if (k + 1u >= win) return;  // (win == 0: an earlier drain's capture, which this drain does not replace)
  if (kind == kOpResult) {
    if (!((arg & kHcBits) || (rem && (arg & AM_F_REMEDY_PENDING)))) return;
    if (((arg ^ ops[win - 1u].y) & kCallTagMask) == 0u) {  // an entry of the winner's own call, or one 2^22·m ops before
      if (!calls) return;
      uint32_t lo = 0, hi = n_calls;  // the first call that starts after op k
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (calls[mid] <= k) lo = mid + 1u;
        else hi = mid;
      }
      if (lo == n_calls || calls[lo] >= win) return;  // (the winner is op win - 1)
    }
  }
  start[i] = kNotInFlight;
}

// Spec updates (am_sweep_update_spec), after apply_state_ops_kernel and store_wf_timeout_kernel: the slot's latest one,
// unless a later upsert or remove replaced the record, rewrites the spec columns of a live slot on top of whatever that
// upsert left, and keeps its status.  Only columns that change are stored, and only a change of masks, kind or zone marks
// the segment for build_planes_dirty_kernel: a status echo with an unchanged spec costs the gathers alone.  `wf` (the
// timeout state, NULL without it) takes the record's wf_timeout for the slot's next run.  Status changes (`chg` NULL
// without tracking): an update that makes a slot with posted results live (NO_RESOURCE or HOST_FALLBACK -> a kind the
// sweep evaluates) hands them to the coming tick, which applies them; if its bit is clear (a list dropped it while the
// slot was not live) it is set, with the pair a pass that finds the bit clear starts from (`det_*` NULL without
// details).  Otherwise the bits and the pairs are left alone.
__global__ void apply_spec_ops_kernel(DevCols c, const uint32_t* __restrict__ marks, const uint32_t* __restrict__ spec_marks,
                                      const uint2* __restrict__ ops, const am_record_t* __restrict__ recs, uint32_t n,
                                      uint32_t* seg_dirty, int32_t* wf, uint32_t* chg, uint8_t* det_applied,
                                      int64_t* det_start, uint32_t* due, int64_t due_epoch) {
  pdl_wait();  // (launched with programmatic stream serialisation: nothing of the predecessor is touched before this)
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 op = ops[k];
  const uint32_t i = op.x, arg = op.y;
  if ((arg & kOpKindMask) != kOpSpec || spec_marks[i] != k + 1u || mark(marks, i, kMarkState) > k + 1u) return;
  const uint32_t f = c.flags[i];
  if (f & AM_F_TOMBSTONE) return;
  const am_record_t& r = recs[arg & ~kOpKindMask];
  uint32_t g = (f & ~(uint32_t)AM_F_SPEC_MASK) | (r.flags & (uint32_t)AM_F_SPEC_MASK);
  if ((f & AM_KIND_MASK) != AM_KIND_STOPPED || (g & AM_KIND_MASK) != AM_KIND_STOPPED) g &= ~AM_F_STOPPED_REPORTED;
  bool planes = ((f ^ g) & (AM_KIND_MASK | AM_F_TZ_MASK)) != 0;
  if (g != f) c.flags[i] = g;
  const uint64_t m[5] = {r.minute, r.hour, r.dom, r.month, r.dow};
  uint64_t* col[5] = {c.minute, c.hour, c.dom, c.month, c.dow};
#pragma unroll
  for (int x = 0; x < 5; ++x)
    if (col[x][i] != m[x]) { col[x][i] = m[x]; planes = true; }
  if (c.ras[i] != r.ras) {
    c.ras[i] = r.ras;
    if (due) due[i] = due_word(r.ras, c.finished_at[i], due_epoch);
  }
  if (c.runs_limit[i] != r.runs_limit) c.runs_limit[i] = r.runs_limit;
  if (c.reset_interval[i] != r.reset_interval) c.reset_interval[i] = r.reset_interval;
  if (wf && wf[i] != r.wf_timeout) wf[i] = r.wf_timeout;
  if (planes) seg_dirty[i / kRecPerWarp] = 1u;
  const uint32_t b = 1u << (i & 31u);
  if (chg && is_live(g) && (g & kPendBits) && !(chg[i / 32u] & b)) {  // (this thread alone owns slot i's bit here)
    if (det_applied) {
      det_applied[i] = (uint8_t)applied_of(g);
      det_start[i] = kNotInFlight;
    }
    atomicOr(chg + i / 32u, b);
  }
}

// The expiry pass's timed-out runs (before note_slots_kernel sets their bits): the timeout's Failed and its run's start.
__global__ void capture_timeouts_kernel(uint8_t* applied, int64_t* start, const uint32_t* __restrict__ bits,
                                        const uint32_t* __restrict__ idx, const int64_t* __restrict__ since,
                                        const uint32_t* __restrict__ count) {
  pdl_wait();  // (launched with programmatic stream serialisation: expire_runs_kernel writes the list)
  const uint32_t n = *count;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const uint32_t i = idx[k];
    const int64_t s = since[k];
    const uint32_t before = ((bits[i / 32u] >> (i & 31u)) & 1u) ? applied[i] : 0u;
    applied[i] = (uint8_t)(before | (is_remedy_run(s) ? AM_CHG_REMEDY_FAILED | AM_CHG_REMEDY_TIMED_OUT
                                                      : AM_CHG_FAILED | AM_CHG_TIMED_OUT));
    start[i] = s;
  }
}

// After the sweep, before note_exceptions_kernel, one warp per tile: a slot the sweep alone adds to the list (STOPPED,
// or in closed loop a completed submission) whose bit is clear starts from (0, kNotInFlight).
__global__ void capture_sweep_kernel(uint8_t* applied, int64_t* start, const uint32_t* __restrict__ bits, const TickOut out,
                                     uint32_t n_tiles, bool closed) {
  pdl_wait();  // (launched with programmatic stream serialisation: the sweep writes the exceptions)
  const int lane = threadIdx.x & 31;
  const uint32_t tile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (tile >= n_tiles) return;  // warp-uniform
  const size_t w0 = (size_t)tile * kTileWords;
  if (closed) {
    for (uint32_t m = out.bitmap[w0 + lane] & ~bits[w0 + lane]; m; m &= m - 1u) {
      const size_t i = (w0 + lane) * 32u + (uint32_t)__ffs((int)m) - 1u;
      applied[i] = 0;
      start[i] = kNotInFlight;
    }
  }
  const uint32_t ne = out.tile_exc[tile];
  for (uint32_t e = (uint32_t)lane; e < ne; e += 32u) {
    const uint32_t x = out.exc_seg[(size_t)tile * kTile + e];
    const size_t i = (size_t)tile * kTile + exc_offset(x);
    if ((exc_action(x) & AM_ACT_STOPPED) && !((bits[i / 32u] >> (i & 31u)) & 1u)) {
      applied[i] = 0;
      start[i] = kNotInFlight;
    }
  }
}

// Turning details on (every slot), am_sweep_load_range (its range) and the end of am_sweep_run_ticks: the pair from the
// flags as they stand, with no start (results pending from before report none).
__global__ void seed_details_kernel(uint8_t* applied, int64_t* start, const uint32_t* __restrict__ flags, uint64_t first,
                                    uint64_t n) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
    applied[first + k] = (uint8_t)applied_of(flags[first + k]);
    start[first + k] = kNotInFlight;
  }
}

// After list_changes_kernel: the pair of every listed slot, by list entry, so that the drains of later calls (which
// capture for the next tick) leave the list's details as the tick left them.  Grid-stride: the count is known on the
// device only.
__global__ void snapshot_details_kernel(const uint32_t* __restrict__ list, const unsigned long long* __restrict__ count,
                                        const uint8_t* __restrict__ applied, const int64_t* __restrict__ start,
                                        uint8_t* e_applied, int64_t* e_start) {
  pdl_wait();  // (launched with programmatic stream serialisation: list_changes_kernel writes the list)
  const uint32_t n = (uint32_t)*count;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const uint32_t i = list[k];
    e_applied[k] = applied[i];
    e_start[k] = start[i];
  }
}

// am_sweep_last_change_details: the details of list entries [0, n) (slots idx, pairs e_applied / e_start) of the tick
// whose output is `out`.  The action is the slot's exception (a binary search of its tile's ascending exceptions), else
// SUBMIT_HC from the bitmap.
__global__ void gather_details_kernel(const uint32_t* __restrict__ idx, uint32_t n, const uint8_t* __restrict__ e_applied,
                                      const int64_t* __restrict__ e_start, const TickOut out, bool closed, int64_t T,
                                      am_change_detail_t* dst) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = idx[k], tile = i / (uint32_t)kTile, off = i % (uint32_t)kTile;
  uint32_t act = ((out.bitmap[i / 32u] >> (i & 31u)) & 1u) ? AM_ACT_SUBMIT_HC : 0u;
  const uint32_t* e = out.exc_seg + (size_t)tile * kTile;
  uint32_t lo = 0, hi = out.tile_exc[tile];
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2u;
    if (exc_offset(e[mid]) < off) lo = mid + 1u;
    else hi = mid;
  }
  if (lo < out.tile_exc[tile] && exc_offset(e[lo]) == off) act = exc_action(e[lo]);
  uint32_t a = e_applied[k];
  const int64_t w = e_start[k];
  am_change_detail_t d;
  d.started = (a & (AM_CHG_SUCCEEDED | AM_CHG_FAILED)) && w != kNotInFlight && !is_remedy_run(w) ? w : kNotInFlight;
  d.remedy_started =
      (a & (AM_CHG_REMEDY_SUCCEEDED | AM_CHG_REMEDY_FAILED)) && is_remedy_run(w) ? run_start(w) : kNotInFlight;
  if (act & AM_ACT_STOPPED) a |= AM_CHG_STOPPED;
  if (closed && (act & AM_ACT_SUBMIT_HC)) {
    a |= AM_CHG_CLOSED_LOOP;
    d.started = T;
  }
  d.applied = a;
  d.action = act;
  dst[k] = d;
}

// am_sweep_read by index and am_sweep_last_changes: the requested columns of the listed slots idx[0..n), column-major
// into dst[c] (blockIdx.y = c).
struct GatherCols {
  const void* src[16];
  void* dst[16];
  uint32_t elem[16];  // 4 or 8 bytes
};
__global__ void gather_columns_kernel(const GatherCols g, const uint32_t* __restrict__ idx, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t c = blockIdx.y, i = idx[k];
  if (g.elem[c] == 8u) ((uint64_t*)g.dst[c])[k] = ((const uint64_t*)g.src[c])[i];
  else ((uint32_t*)g.dst[c])[k] = ((const uint32_t*)g.src[c])[i];
}

}  // namespace amsweep

#include "sweep_block.cuh"
