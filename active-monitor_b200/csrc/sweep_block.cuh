// sweep_block.cuh — K consecutive one-second ticks per pass over the columns ("temporal blocking",
// SURVEY §7 step 9; the timer-wheel reading of §8f-1 / hcc.go:751).
//
// am_sweep_run_ticks streams seconds back to back (BASELINE config 5: one simulated day = 86 400 ticks).
// With one sweep per tick every tick re-reads 16..56 B per record to find the ~4 % that are due.  But
// nothing reaches a record from outside between the ticks of such a run, so its whole future inside a
// block of K ticks (96 by default) follows from its own columns: this kernel loads a record ONCE, then steps it from
// event to event in registers — the reference's own shape, a timer per HealthCheck (time.AfterFunc,
// hcc.go:751) instead of a scan per second:
//
//   interval / "@every" check   next event = finishedAt + repeatAfterSec (hcc.go:264), every tick while no
//                               timer is armed (controller restart, hcc.go:161)
//   5-field cron                next event = the next tick whose LOCAL second is 0 (robfig activates on
//                               the minute; the zone's offset decides which UTC second that is)
//   parse error                 every tick (hcc.go:254-257: warning + requeue)
//   stopped                     once (hcc.go:238-250)
//   posted result / carry bits  the first tick of the block
//
// and at an event tick evaluates EXACTLY what sweep_tick_kernel evaluates for that (record, tick) —
// interval_due and is_interval_kind for the schedule ladder, result_step for the posted result and the
// closed-loop completion, load_state / store_changed_state for the remedy and counter columns — so the
// per-tick statistics and the columns after the block are bit-identical to K single ticks (tests:
// run_ticks blocked == unblocked == oracle).  Work is O(events), not O(records x ticks); the columns are
// read and written once per K ticks.  What it does NOT produce is the per-tick (index, action) lists: a run of ticks publishes
// per-tick statistics (counts, action counts, index checksums — am_tick_stats_t), which is all
// am_sweep_run_ticks ever returned to the host.  Reported separately from the K = 1 roofline number.
//
// SIM (am_sweep_simulate): the same walk with the hold in flight, the remedy hold and workflow timeouts on, and every
// held run ending at its simulated end (sim_run_end).  The record's run is one more thing carried in registers: its
// since word (start and kind), its end C and its deadline D.  While the run is held the record's next event is
// min(C, D); its cron minutes and interval timers are suppressed, because a held check is never submitted.  At an event
// tick the record takes the simulated post, then the expiry, then exactly what the hold variants of sweep_tick_kernel
// evaluate; a run that starts sets since (and D = T + W), and the record resumes its schedule when the run ends.
#pragma once

#include <type_traits>

namespace amsweep {

#ifndef AM_BLOCK_MAX_TICKS
#define AM_BLOCK_MAX_TICKS 128
#endif
constexpr int kMaxBlockTicks = AM_BLOCK_MAX_TICKS;
constexpr int kDefaultBlockTicks = 96;  // faster per tick than 64 or 128 (10 M records, config 5)
#ifndef AM_BLOCK_THREADS
#define AM_BLOCK_THREADS 128
#endif
constexpr int kBlockThreads = AM_BLOCK_THREADS;
// Occupancy is what this kernel wants: its warps wait on each other (per-class lists of different lengths, one
// barrier before the flush) and on shared atomics.  256 threads at 94 registers = 2 CTAs per SM spent half of its
// stall samples at the final barrier; 128 threads capped at 64 registers (8 CTAs per SM, a few bytes of spills) was
// much faster, and 256 threads / 4 CTAs at the same cap faster still.
#ifndef AM_BLOCK_MIN_CTAS
#define AM_BLOCK_MIN_CTAS 8
#endif
constexpr int kBlockRecords = 4 * kBlockThreads;  // four consecutive records per thread in the classification pass
constexpr int kBlockClasses = 4;                  // by expected number of events in the block: <= 2, <= 8, <= 24, more

struct BlockParams {
  DevCols c;
  uint64_t n_records, shard_base, seed;
  int64_t T0;                  // first tick of the block
  uint32_t K;                  // ticks in the block, <= kMaxBlockTicks
  const int32_t* tz_off;       // per-zone UTC offsets valid for the whole block (NULL: no zone registered)
  unsigned long long* stats;   // K rows of 16 accumulators (am_tick_stats_t layout), zero on entry
};

// SIM: the run state of every slot and the simulation's draws
struct SimBlockParams : BlockParams {
  int64_t* since;                    // [cap] the hold's since words (both kinds of run)
  int64_t* deadline;                 // [cap] deadlines; NULL without timeout state (then nothing times out)
  const int32_t* wf_timeout;         // [cap] the slots' workflow timeouts; NULL without timeout state
  unsigned long long* seg_deadline;  // [cap / kRecPerWarp] expire_runs_kernel's bounds: lowered for the deadlines set
  SimDraw q;
  unsigned long long* sim;           // K rows of 4 accumulators (am_sim_tick_t layout), zero on entry
};

// first tick index u > t at which the LOCAL second (UTC + off) is 0
__device__ __forceinline__ int64_t next_local_minute(int64_t T0, int64_t t, int32_t off) {
  int64_t m = (T0 + t + 1 + (int64_t)off) % 60;
  if (m < 0) m += 60;
  return t + 1 + (m ? 60 - m : 0);
}

// Per-CTA statistics of a block of ticks, in shared memory.
struct BlockStats {
  uint32_t cnt[kMaxBlockTicks][13];   // [0] emitted, [1..8] action bits, [9..12] results applied
  uint32_t sum[kMaxBlockTicks];       // sum of CTA-local offsets of the emitted records
  uint32_t x[kMaxBlockTicks][2];      // xor of the emitted global indices
  // records that emit the same bare action on EVERY tick from some tick on (a parse error: hcc.go:254-257
  // warns on every pass; an open-loop check that stays due): registered once, as a delta at their first
  // such tick, and integrated over the ticks when the CTA flushes.  [.][0] = SUBMIT_HC, [.][1] = PARSE_ERROR
  uint32_t c_cnt[kMaxBlockTicks][2], c_sum[kMaxBlockTicks][2], c_x[kMaxBlockTicks][2][2];
  uint16_t list[kBlockClasses][kBlockRecords];  // records with events, by class
  uint32_t n_list[kBlockClasses];
};
// SIM: per tick and kind of run (health check, remedy) the change in the number of held runs (+1 at a start, -1 at an
// end; a run held at the block's start counts as a start at tick 0), integrated over the ticks at the flush as the
// constant emitters are, and the runs the tick timed out
struct SimBlockStats : BlockStats {
  uint32_t run_d[kMaxBlockTicks][2];  // (modulo 2^32: -1 is 0xFFFFFFFF)
  uint32_t run_to[kMaxBlockTicks][2];
};

// a since word's kind of run, as the index of the per-kind rows
__device__ __forceinline__ int sim_kind(int64_t since) { return is_remedy_run(since) ? 1 : 0; }

__device__ __forceinline__ void block_constant(BlockStats& S, int which, int64_t t_from, int64_t K, uint64_t g, uint32_t loc) {
  if (t_from >= K) return;
  atomicAdd(&S.c_cnt[t_from][which], 1u);
  atomicAdd(&S.c_sum[t_from][which], loc);
  atomicXor(&S.c_x[t_from][which][0], (uint32_t)g);
  atomicXor(&S.c_x[t_from][which][1], (uint32_t)(g >> 32));
}

// One record through the block, event by event (see the header of this file).
template <bool CLOSED, bool SIM = false, class Params = BlockParams, class Stats = BlockStats>
__device__ __forceinline__ void block_record(const Params& p, Stats& S, uint64_t cta_base, uint32_t loc) {
  const int64_t K = (int64_t)p.K;
  const uint64_t i = cta_base + loc;
  const uint64_t g = p.shard_base + i;
  uint32_t f = ld_stream(p.c.flags + i);
  const int32_t rasv = ld_stream(p.c.ras + i);
  int64_t fa = ld_stream(p.c.finished_at + i);
  const uint32_t kind = f & AM_KIND_MASK;
  const bool is_iv = is_interval_kind(kind);
  const bool is_cron = kind == AM_KIND_CRON_SPEC;
  int32_t zoff = 0;
  uint64_t mi = 0, hr = 0, dm = 0, mo = 0, dw = 0;
  if (is_cron) {
    const uint32_t tz = f >> AM_F_TZ_SHIFT;
    if (tz && p.tz_off) zoff = p.tz_off[tz];
    mi = ld_stream(p.c.minute + i); hr = ld_stream(p.c.hour + i); dm = ld_stream(p.c.dom + i);
    mo = ld_stream(p.c.month + i); dw = ld_stream(p.c.dow + i);
  }
  // remedy / counter state: every due record needs it in closed loop, a posted result in open loop (SIM: any result)
  RecState s{};
  const bool with_state = CLOSED || SIM || (f & kPendBits) != 0;
  if (with_state) load_state(p.c, i, s);
  const RecState s0 = s;
  const uint32_t f0 = f;
  const int64_t fa0 = fa;

  // SIM: the run.  sv = since, D = deadline, C = the held run's simulated end (INT64_MAX while none is held), W = the
  // slot's workflow timeout.  A record that is not live keeps its run until it ends and is never evaluated.
  int64_t sv = kNotInFlight, D = kNoDeadline, C = INT64_MAX;
  uint32_t cbits = 0;
  int32_t W = 0;
  const bool live = !SIM || is_live(f);
  auto held = [&] { return sv != kNotInFlight && sv >= fa && !(f & kHcBits); };  // held_run on the registers
  auto set_end = [&] {
    if constexpr (SIM) C = held() ? sim_run_end(p.q, g, sv, f, &cbits) : INT64_MAX;
  };
  // the held-run rows after tick t: the record's change against `was` / `was_kind`, the state before the tick
  auto note_run = [&](int64_t t, bool was, int was_kind) {
    if constexpr (SIM) {
      const bool now = held();
      if (was && (!now || sim_kind(sv) != was_kind)) atomicAdd(&S.run_d[t][was_kind], 0xFFFFFFFFu);
      if (now && (!was || sim_kind(sv) != was_kind)) atomicAdd(&S.run_d[t][sim_kind(sv)], 1u);
      set_end();
    }
  };
  if constexpr (SIM) {
    sv = p.since[i];
    if (p.deadline) {
      D = p.deadline[i];
      W = p.wf_timeout[i];
    }
    set_end();
    if (held()) atomicAdd(&S.run_d[0][sim_kind(sv)], 1u);
  }
  const int64_t sv0 = sv, D0 = D;

  auto plain_event = [&](int64_t t) -> int64_t {  // the first tick index > t at which this record can act
    if (kind == AM_KIND_PARSE_ERROR) return t + 1;
    if (kind == AM_KIND_STOPPED) return (f & AM_F_STOPPED_REPORTED) ? K : t + 1;
    if (is_iv) {
      if (!(f & AM_F_TIMER_ARMED)) return t + 1;  // no timer: the reference submits on every pass
      const int64_t d = fa + (int64_t)rasv - p.T0;  // elapsed >= ras  <=>  tick index >= d
      return d > t + 1 ? d : t + 1;
    }
    return next_local_minute(p.T0, t, zoff);  // 5-field schedule
  };
  auto next_event = [&](int64_t t) -> int64_t {
    if constexpr (SIM) {  // the run's next event, min(C, D); a held check's schedule is suppressed
      int64_t e = held() ? C - p.T0 : K;
      if (D != kNoDeadline && D - p.T0 < e) e = D - p.T0;
      if (e < t + 1) e = t + 1;
      if (!live || (held() && (is_iv || is_cron))) return e;
      const int64_t u = plain_event(t);
      return u < e ? u : e;
    }
    return plain_event(t);
  };

  int64_t t = (live && (f & (kPendBits | AM_F_CARRY_MASK))) ? 0 : next_event(-1);
  while (t < K) {
    const int64_t T = p.T0 + t;
    bool was = false;
    int was_kind = 0;
    if constexpr (SIM) {
      was = held();
      was_kind = sim_kind(sv);
      if (was && C <= T) {  // the simulated post: the drain of am_sweep_post_result (clear_since_kernel)
        f = sim_post(f, cbits);
        sv = kNotInFlight;
      }
      if (D <= T) {  // the expiry pass (expire_runs_kernel)
        D = kNoDeadline;
        if (live && held()) {
          f = is_remedy_run(sv) ? ((f & ~AM_F_REMEDY_OUTCOME_OK) | AM_F_REMEDY_PENDING) : (f | AM_F_PENDING_FAIL);
          atomicAdd(&S.run_to[t][sim_kind(sv)], 1u);
          sv = kNotInFlight;
        }
      }
      if (!live) {
        note_run(t, was, was_kind);
        t = next_event(t);
        continue;
      }
    }
    // ---- exactly sweep_tick_kernel's decision for (record, T) ----
    const bool pending = (f & kPendBits) != 0;
    const bool due_iv = interval_due(f, rasv, fa, T);
    bool due_cron = false;
    if (is_cron) {
      const TickWords w = tick_words_from_unix(T + (int64_t)zoff);
      due_cron = cron_matches(w, mi, hr, dm, mo, dw);
    }
    const bool due = is_iv ? due_iv : (is_cron && due_cron);
    const bool stopped_now = kind == AM_KIND_STOPPED && !(f & AM_F_STOPPED_REPORTED);
    uint32_t act = (due ? AM_ACT_SUBMIT_HC : 0u) | (stopped_now ? AM_ACT_STOPPED : 0u) |
                   (kind == AM_KIND_PARSE_ERROR ? AM_ACT_PARSE_ERROR : 0u);
    if constexpr (SIM) {  // the hold (HOLD / TIMEOUT variants): a held check is not submitted, a submitted one runs
      if (due) {
        if (held()) {
          act &= ~AM_ACT_SUBMIT_HC;
        } else {
          sv = T;
          if (p.deadline) D = W > 0 ? T + W : kNoDeadline;
        }
      }
    }
    if (f & AM_F_CARRY_MASK) {
      act |= carried_actions(f);
      f &= ~AM_F_CARRY_MASK;
    }
    if (stopped_now) {  // hcc.go:238-250
      f |= AM_F_STOPPED_REPORTED;
      fa = T;
    }
    uint32_t res = 0;
    if (pending || (CLOSED && due)) {
      s.flags = f;
      s.fa = fa;
      const uint32_t a = result_step<CLOSED>(s, T, due, p.seed, g, res);
      act |= a;
      if constexpr (SIM) {  // the remedy hold (REMEDY variants): start_remedy_run
        if (starts_remedy_run(a, f)) {
          sv = T + kRemedyRun;
          if (p.deadline) D = W > 0 ? T + W : kNoDeadline;
          act &= ~AM_ACT_SUBMIT_HC;
        }
      }
      f = s.flags;
      fa = s.fa;
    }
    // ---- this tick's statistics (what expand_kernel derives from the emitted list) ----
    if (act) {
      atomicAdd(&S.cnt[t][0], 1u);
      uint32_t bits = act;
      while (bits) {
        const int b = __ffs((int)bits) - 1;
        bits &= bits - 1u;
        atomicAdd(&S.cnt[t][1 + b], 1u);
      }
      atomicXor(&S.x[t][0], (uint32_t)g);
      atomicXor(&S.x[t][1], (uint32_t)(g >> 32));
      atomicAdd(&S.sum[t], loc);
    }
    if (res) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if ((res >> (8 * q)) & 0xFFu) atomicAdd(&S.cnt[t][9 + q], (res >> (8 * q)) & 0xFFu);
    }
    if constexpr (SIM) note_run(t, was, was_kind);
    // from here on the same bare action on every tick, and nothing changes any more?  (SIM: a due check is submitted
    // and held; a parse error with a run or a deadline left still has events)
    if (kind == AM_KIND_PARSE_ERROR && (!SIM || (!held() && D == kNoDeadline))) { block_constant(S, 1, t + 1, K, g, loc); break; }
    if (!SIM && !CLOSED && is_iv && due) { block_constant(S, 0, t + 1, K, g, loc); break; }  // stays due: nothing completes it in open loop
    t = next_event(t);
  }

  // ---- write back what changed ----
  if (f != f0) st_stream(p.c.flags + i, f);
  if (fa != fa0) st_stream(p.c.finished_at + i, fa);
  if (with_state) store_changed_state(p.c, i, s, s0);
  if constexpr (SIM) {  // once per block; expire_runs_kernel's bound stays a lower bound of the deadlines
    if (sv != sv0) p.since[i] = sv;
    if (D != D0) {
      p.deadline[i] = D;
      if (D != kNoDeadline) atomicMin(p.seg_deadline + i / (uint64_t)kRecPerWarp, biased_key(D));
    }
  }
}

// SIM, pass 1: the expected number of events of a record in the block (0: not listed).  A record whose held run
// neither ends nor meets its deadline inside the block and that has nothing else to do is registered once as held
// for the whole block; a parse error with no run event is a constant emitter, as without SIM.
__device__ __forceinline__ int64_t sim_events(const SimBlockParams& p, SimBlockStats& S, uint32_t loc, uint64_t g,
                                              uint32_t f, int32_t rasv, int64_t fa, int64_t sv, int64_t D) {
  const int64_t K = (int64_t)p.K;
  const uint32_t kind = f & AM_KIND_MASK;
  const bool hd = sv != kNotInFlight && sv >= fa && !(f & kHcBits);
  int64_t e = K;  // the run's first event
  if (hd) {
    uint32_t bits;
    e = sim_run_end(p.q, g, sv, f, &bits) - p.T0;
  }
  if (D != kNoDeadline && D - p.T0 < e) e = D - p.T0;
  const bool run_ev = e < K;
  int64_t n_ev = run_ev ? 2 : 0;
  const bool first_tick = (f & (kPendBits | AM_F_CARRY_MASK)) != 0;
  if (!is_live(f)) {
  } else if (kind == AM_KIND_PARSE_ERROR) {
    if (!first_tick && !run_ev) {
      block_constant(S, 1, 0, K, g, loc);
    } else {
      n_ev = K;
    }
  } else if (kind == AM_KIND_STOPPED) {
    n_ev += (first_tick || !(f & AM_F_STOPPED_REPORTED)) ? 1 : 0;
  } else if (hd && !run_ev && !first_tick) {
    // a held check: its schedule is suppressed for the whole block
  } else if (kind == AM_KIND_CRON_SPEC) {
    int32_t zoff = 0;
    const uint32_t tz = f >> AM_F_TZ_SHIFT;
    if (tz && p.tz_off) zoff = p.tz_off[tz];
    const int64_t m0 = next_local_minute(p.T0, -1, zoff);
    n_ev += (first_tick ? 1 : 0) + (m0 < K ? 1 + (K - 1 - m0) / 60 : 0);
  } else {  // INTERVAL / CRON_EVERY
    const int64_t step = rasv > 0 ? (int64_t)rasv : 1;
    if (!(f & AM_F_TIMER_ARMED) || first_tick) {
      n_ev += 1 + (K - 1) / step;
    } else {
      int64_t d = fa + (int64_t)rasv - p.T0;
      if (d < 0) d = 0;
      if (d < K) n_ev += 1 + (K - 1 - d) / step;
    }
  }
  if (n_ev <= 0 && hd) atomicAdd(&S.run_d[0][sim_kind(sv)], 1u);
  return n_ev;
}

template <bool CLOSED, bool SIM = false>
__global__ void __launch_bounds__(kBlockThreads, AM_BLOCK_MIN_CTAS)
    sweep_block_kernel(const std::conditional_t<SIM, SimBlockParams, BlockParams> p) {
  __shared__ std::conditional_t<SIM, SimBlockStats, BlockStats> S;
  const int tid = threadIdx.x;
  {
    uint32_t* z = reinterpret_cast<uint32_t*>(&S);
    constexpr int kZero = (int)(offsetof(BlockStats, list) / 4);  // everything before the lists
    for (int k = tid; k < kZero; k += kBlockThreads) z[k] = 0;
    if (tid < kBlockClasses) S.n_list[tid] = 0;
    if constexpr (SIM) {  // ... and the run rows
      uint32_t* r = reinterpret_cast<uint32_t*>(&S.run_d[0][0]);
      for (int k = tid; k < 4 * kMaxBlockTicks; k += kBlockThreads) r[k] = 0;
    }
  }
  __syncthreads();

  const uint64_t cta_base = (uint64_t)blockIdx.x * kBlockRecords;
  const int64_t K = (int64_t)p.K;

  // ---- pass 1: classify.  16 B per record (flags, repeatAfterSec, finishedAt), four records per thread (SIM: 16 B
  //      more, since and deadline).
  //      Records that cannot act inside the block — the majority: an armed timer that fires later — cost
  //      nothing more; records that emit the same action on every tick are registered as constants;
  //      the others go onto a list by their expected number of events, so that the lanes of a warp of
  //      pass 2 run loops of similar length (per-lane ownership ran at 4 of 32 lanes active: one
  //      "@every 500ms" check keeps its lane busy for 64 events while its neighbours have none).
  {
    const uint32_t loc0 = 4u * (uint32_t)tid;
    const uint64_t i0 = cta_base + loc0;  // columns are padded to whole tiles; slots past n_records are tombstones
    const uint4 f4 = ld_stream(reinterpret_cast<const uint4*>(p.c.flags + i0));
    const int4 r4 = ld_stream(reinterpret_cast<const int4*>(p.c.ras + i0));
    const longlong2 a01 = ld_stream(reinterpret_cast<const longlong2*>(p.c.finished_at + i0));
    const longlong2 a23 = ld_stream(reinterpret_cast<const longlong2*>(p.c.finished_at + i0 + 2));
    longlong2 s01{}, s23{}, d01{}, d23{};
    if constexpr (SIM) {
      s01 = ld_stream(reinterpret_cast<const longlong2*>(p.since + i0));
      s23 = ld_stream(reinterpret_cast<const longlong2*>(p.since + i0 + 2));
      d01 = d23 = make_longlong2(kNoDeadline, kNoDeadline);
      if (p.deadline) {
        d01 = ld_stream(reinterpret_cast<const longlong2*>(p.deadline + i0));
        d23 = ld_stream(reinterpret_cast<const longlong2*>(p.deadline + i0 + 2));
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t f = q == 0 ? f4.x : q == 1 ? f4.y : q == 2 ? f4.z : f4.w;
      const int32_t rasv = q == 0 ? r4.x : q == 1 ? r4.y : q == 2 ? r4.z : r4.w;
      const int64_t fa = q == 0 ? a01.x : q == 1 ? a01.y : q == 2 ? a23.x : a23.y;
      const uint32_t loc = loc0 + (uint32_t)q;
      if constexpr (SIM) {
        const int64_t sv = q == 0 ? s01.x : q == 1 ? s01.y : q == 2 ? s23.x : s23.y;
        const int64_t D = q == 0 ? d01.x : q == 1 ? d01.y : q == 2 ? d23.x : d23.y;
        const int64_t n_ev = sim_events(p, S, loc, p.shard_base + cta_base + loc, f, rasv, fa, sv, D);
        if (n_ev <= 0) continue;
        const int c = n_ev <= 2 ? 0 : (n_ev <= 8 ? 1 : (n_ev <= 24 ? 2 : 3));
        S.list[c][atomicAdd(&S.n_list[c], 1u)] = (uint16_t)loc;
        continue;
      }
      const uint32_t kind = f & AM_KIND_MASK;
      if (!is_live(f)) continue;  // tombstones, NO_RESOURCE (hcc.go:227), host-fallback: never evaluated
      const bool first_tick = (f & (kPendBits | AM_F_CARRY_MASK)) != 0;  // posted result / carried action: tick 0
      const uint64_t g = p.shard_base + cta_base + loc;
      int64_t n_ev = 0;  // expected events in the block (an upper bound is fine: it only picks the list)
      if (kind == AM_KIND_PARSE_ERROR) {
        if (!first_tick) { block_constant(S, 1, 0, K, g, loc); continue; }
        n_ev = 1;
      } else if (kind == AM_KIND_STOPPED) {
        n_ev = (first_tick || !(f & AM_F_STOPPED_REPORTED)) ? 1 : 0;
      } else if (kind == AM_KIND_CRON_SPEC) {
        int32_t zoff = 0;
        const uint32_t tz = f >> AM_F_TZ_SHIFT;
        if (tz && p.tz_off) zoff = p.tz_off[tz];
        const int64_t m0 = next_local_minute(p.T0, -1, zoff);
        n_ev = (first_tick ? 1 : 0) + (m0 < K ? 1 + (K - 1 - m0) / 60 : 0);
      } else {  // INTERVAL / CRON_EVERY
        const int64_t step = rasv > 0 ? (int64_t)rasv : 1;
        if (!(f & AM_F_TIMER_ARMED) || first_tick) {
          if (!CLOSED && !first_tick) { block_constant(S, 0, 0, K, g, loc); continue; }  // due on every tick, nothing changes
          n_ev = 1 + (K - 1) / step;
        } else {
          int64_t d = fa + (int64_t)rasv - p.T0;
          if (d < 0) d = 0;
          if (d >= K) continue;  // its timer fires after the block
          if (!CLOSED) { block_constant(S, 0, d, K, g, loc); continue; }  // due from tick d on
          n_ev = 1 + (K - 1 - d) / step;
        }
      }
      if (n_ev <= 0) continue;
      const int c = n_ev <= 2 ? 0 : (n_ev <= 8 ? 1 : (n_ev <= 24 ? 2 : 3));
      S.list[c][atomicAdd(&S.n_list[c], 1u)] = (uint16_t)loc;
    }
  }
  __syncthreads();
  // (Measured and dropped: a second kernel for the longest loops, run in full warps — slower, its lanes
  //  all sit on the same tick and collide on every shared atomic; grouping the lanes of a warp by tick
  //  with match.any + redux before the atomics, and 128-thread CTAs — slower still:
  //  the collectives cost more than the conflicts they remove.)

  // ---- pass 2: the listed records, longest loops first; the warps start at different places so that the
  //      (short) head of every list does not always land on warp 0
#pragma unroll 1
  for (int c = kBlockClasses - 1; c >= 0; --c) {
    const uint32_t n = S.n_list[c];
    for (uint32_t k = ((uint32_t)tid + (uint32_t)(kBlockThreads / 4) * (uint32_t)c) & (kBlockThreads - 1); k < n; k += kBlockThreads)
      block_record<CLOSED, SIM>(p, S, cta_base, S.list[c][k]);
  }
  __syncthreads();

  // ---- integrate the constant emitters over the ticks (thread t: everything registered at ticks <= t)
  for (int t = tid; t < (int)p.K; t += kBlockThreads) {
    uint32_t c0 = 0, c1 = 0, s0 = 0, s1 = 0, x0 = 0, x1 = 0;
    for (int u = 0; u <= t; ++u) {
      c0 += S.c_cnt[u][0]; c1 += S.c_cnt[u][1];
      s0 += S.c_sum[u][0]; s1 += S.c_sum[u][1];
      x0 ^= S.c_x[u][0][0] ^ S.c_x[u][1][0];
      x1 ^= S.c_x[u][0][1] ^ S.c_x[u][1][1];
    }
    S.cnt[t][0] += c0 + c1;
    S.cnt[t][1] += c0;      // AM_ACT_SUBMIT_HC   (bit 0)
    S.cnt[t][4] += c1;      // AM_ACT_PARSE_ERROR (bit 3)
    S.sum[t] += s0 + s1;
    S.x[t][0] ^= x0;
    S.x[t][1] ^= x1;
  }
  __syncthreads();

  // ---- CTA -> global: one RED per non-zero (tick, field) ----
  const unsigned long long gbase = (unsigned long long)(p.shard_base + cta_base);
  for (uint32_t k = (uint32_t)tid; k < p.K * 16u; k += kBlockThreads) {
    const uint32_t t = k >> 4, fld = k & 15u;
    unsigned long long* dst = p.stats + (size_t)t * kNumAcc + fld;
    if (fld >= 1 && fld <= 13) {
      const uint32_t v = S.cnt[t][fld - 1];
      if (v) atomicAdd(dst, (unsigned long long)v);
    } else if (fld == 14) {
      const unsigned long long x = ((unsigned long long)S.x[t][1] << 32) | S.x[t][0];
      if (x) atomicXor(dst, x);
    } else if (fld == 15) {
      const uint32_t cnt = S.cnt[t][0];
      if (cnt) atomicAdd(dst, (unsigned long long)cnt * gbase + S.sum[t]);
    }
  }
  if constexpr (SIM) {  // ---- the run rows: the held runs after tick t (thread t: the changes at ticks <= t), the timed out
    for (int t = tid; t < (int)p.K; t += kBlockThreads) {
      uint32_t h0 = 0, h1 = 0;
      for (int u = 0; u <= t; ++u) {
        h0 += S.run_d[u][0];
        h1 += S.run_d[u][1];
      }
      unsigned long long* row = p.sim + (size_t)t * 4;
      if (h0) atomicAdd(row + 0, (unsigned long long)h0);
      if (h1) atomicAdd(row + 1, (unsigned long long)h1);
      if (S.run_to[t][0]) atomicAdd(row + 2, (unsigned long long)S.run_to[t][0]);
      if (S.run_to[t][1]) atomicAdd(row + 3, (unsigned long long)S.run_to[t][1]);
    }
  }
}

}  // namespace amsweep
