// admission_kernels.cuh — the submit budget (am_sweep_set_submit_budget, DESIGN.md section 6 item 19): after a tick's
// sweep and before scan_groups_kernel, the tick's AM_ACT_SUBMIT_HC entries are cut to the budget IN PLACE in the sweep's
// own output (bitmap, per-tile exceptions, per-group counts), so that the list rebuild, the statistics and the NVLink
// exchange read the admitted list unchanged.
//
// State (allocated at the first finite budget):
//   since[i] of the hold, the admission's own `wait[i]` (the second since which slot i waits for admission, or
//   kNotWaiting) and a FIFO of waiting slots in admission order: by (wait[i], i) ascending.  A FIFO entry is checked
//   lazily against wait[]: removes, loads and posted phases clear wait[] at their drain and leave the entry behind,
//   the next tick drops it.
// One tick (host: launch_admission):
//   adm_masks_kernel   per group: the sweep's SUBMIT_HC records as a bitmap (`sub`), counted per group;
//   adm_check_kernel   per FIFO entry: still waiting?  A candidate?  (one the sweep submitted leaves `sub`);
//   adm_plan_kernel    one CTA: the FIFO's candidate ranks and the fresh candidates' per-group offsets, the cut;
//   adm_fifo_kernel    per FIFO entry: the first `budget` candidates are admitted (added to the list if the sweep did
//                      not submit them), the rest stay and are trimmed from the list if it did;
//   adm_fresh_kernel   per group: fresh candidates past the remaining budget are trimmed and start waiting at T;
//   adm_merge_kernel   the kept FIFO entries and the new ones merged by (second, slot) into the FIFO.
// Every pass is over the bitmap (0.125 B per record), the candidates or the backlog; none reads the columns of a record
// that is neither.
#pragma once
#ifndef AMSWEEP_EMULATE  // tests/emu compiles this file for the CPU (cuda_emu.h supplies the model)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "sweep_kernels.cuh"

namespace amsweep {

constexpr int64_t kNotWaiting = INT64_MIN;
static_assert(kNotWaiting == kNotInFlight, "one 'not in the state' value for every AM_SEL_* state");
constexpr int kAdmBlock = 256;  // threads per CTA of the per-entry passes = FIFO entries per chunk
static_assert(kGroupWords == kAdmBlock, "adm_block_scan serves the per-group passes (one word per thread) as well");

// The admission's device-side counters: the backlog's length and the last tick's numbers (am_admission_t).
struct AdmCtl {
  unsigned long long n_fifo;      // entries in the FIFO (every one still waiting after the tick that wrote it)
  unsigned long long n_def_cand;  // this tick: waiting candidates (D)
  unsigned long long n_fresh;     // ... fresh candidates (F)
  unsigned long long room;        // ... budget left for the fresh ones: max(budget - D, 0)
  unsigned long long n_keep;      // ... waiting candidates not admitted
  unsigned long long n_new;       // ... fresh candidates deferred
  unsigned long long n_candidates, n_admitted, n_deferred;
  long long oldest;
};

struct AdmParams {
  TickOut out;                   // the tick's buffer set, as the sweep left it
  uint32_t n_groups;
  uint32_t n_tiles;
  DevCols c;
  int64_t* since;
  int64_t* deadline;             // NULL without the timeout state
  const int32_t* wf_timeout;     // NULL without the timeout state
  unsigned long long* seg_deadline;
  int64_t* wait;                 // [cap] second since which the slot waits, kNotWaiting
  uint32_t* fifo;                // [cap] waiting slots in admission order
  uint32_t* keep;                // [cap] this tick's waiting candidates that stay, in order
  uint32_t* fresh;               // [cap] this tick's newly deferred slots, ascending
  uint8_t* cand;                 // [cap] per FIFO entry: 0 dropped, 1 candidate, 3 candidate the sweep submitted
  uint32_t* sub;                 // [n_groups * kGroupWords] fresh SUBMIT_HC records
  uint32_t* group_sub;           // [n_groups] fresh SUBMIT_HC records per group, then their exclusive prefix
  uint32_t* chunk;               // [cap / kAdmBlock] candidates per FIFO chunk, then their exclusive prefix
  AdmCtl* ctl;
  unsigned long long budget;
  int64_t T;
};

// The exception entry of record `off` of tile `tile`, or nullptr (its action is the bare SUBMIT_HC, or it has none).
__device__ __forceinline__ uint32_t* adm_exception(const TickOut& o, uint32_t tile, uint32_t off) {
  uint32_t lo = 0, hi = o.tile_exc[tile];
  uint32_t* e = o.exc_seg + (size_t)tile * kTile;
  while (lo < hi) {  // a tile's entries ascend by record
    const uint32_t mid = (lo + hi) / 2;
    if (exc_offset(e[mid]) < off) lo = mid + 1; else hi = mid;
  }
  return lo < o.tile_exc[tile] && exc_offset(e[lo]) == off ? e + lo : nullptr;
}

// Take SUBMIT_HC off slot i's entry (an entry with nothing left leaves the list) and restore the run it started: none.
__device__ __forceinline__ void adm_trim(const AdmParams& a, uint32_t i) {
  if (uint32_t* e = adm_exception(a.out, i / kTile, i % kTile)) {
    *e &= ~AM_ACT_SUBMIT_HC;  // (an exception has another action bit: it stays one)
  } else {
    atomicAnd(&a.out.bitmap[i >> 5], ~(1u << (i & 31)));
    atomicAdd(&a.out.group_count[i / kGroupRecords], 0xFFFFFFFFu);
  }
  a.since[i] = kNotInFlight;
  if (a.deadline) a.deadline[i] = kNoDeadline;
}

// Give slot i's entry SUBMIT_HC (a record with no entry gets one) and start its run at T, as the sweep does.
__device__ __forceinline__ void adm_force(const AdmParams& a, uint32_t i) {
  if (uint32_t* e = adm_exception(a.out, i / kTile, i % kTile)) {
    *e |= AM_ACT_SUBMIT_HC;
  } else {
    atomicOr(&a.out.bitmap[i >> 5], 1u << (i & 31));
    atomicAdd(&a.out.group_count[i / kGroupRecords], 1u);
  }
  a.since[i] = a.T;
  if (a.deadline) {
    const int32_t W = a.wf_timeout[i];
    a.deadline[i] = W > 0 ? a.T + W : kNoDeadline;
    if (W > 0) atomicMin(a.seg_deadline + i / (uint32_t)kRecPerWarp, biased_key(a.T + W));
  }
}

// Block-wide exclusive prefix of v (blockDim.x == kAdmBlock); *total = the block's sum.
__device__ __forceinline__ uint32_t adm_block_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t incl = warp_inclusive_scan(v, lane);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int k = 0; k < kAdmBlock / 32; ++k) {
    before += k < warp ? s_warp[k] : 0u;
    all += s_warp[k];
  }
  __syncthreads();  // (s_warp is reused by the caller's next round)
  *total = all;
  return before + incl - v;
}

// One word per thread, one group per CTA: the group's SUBMIT_HC records (bitmap bits whose exception, if any, has the
// bit) and their count.
__global__ void __launch_bounds__(kGroupWords) adm_masks_kernel(const AdmParams a) {
  __shared__ uint32_t s_m[kGroupWords];
  __shared__ uint32_t s_warp[kGroupWords / 32];
  const uint32_t g = blockIdx.x, t = threadIdx.x;
  const size_t w = (size_t)g * kGroupWords + t;
  s_m[t] = a.out.bitmap[w];
  __syncthreads();
  for (uint32_t k = 0; k < (uint32_t)kGroupTiles; ++k) {
    const uint32_t tile = g * kGroupTiles + k;
    if (tile >= a.n_tiles) break;
    const uint32_t nx = a.out.tile_exc[tile];
    for (uint32_t x = t; x < nx; x += kGroupWords) {
      const uint32_t e = a.out.exc_seg[(size_t)tile * kTile + x];
      if (!(exc_action(e) & AM_ACT_SUBMIT_HC)) {
        const uint32_t off = k * kTile + exc_offset(e);
        atomicAnd(&s_m[off >> 5], ~(1u << (off & 31)));
      }
    }
  }
  __syncthreads();
  const uint32_t m = s_m[t];
  a.sub[w] = m;
  uint32_t total;
  (void)adm_block_scan((uint32_t)__popc(m), s_warp, &total);
  if (t == 0) a.group_sub[g] = total;
}

// Per FIFO entry (chunks of kAdmBlock entries): is its slot still waiting, and a candidate?  A slot the sweep submitted
// is one (its bit leaves `sub`: it is not fresh); otherwise one that is live, can be due and is not held — its waiting
// ends when it is not.
__global__ void __launch_bounds__(kAdmBlock) adm_check_kernel(const AdmParams a) {
  __shared__ uint32_t s_warp[kAdmBlock / 32];
  const uint64_t n = a.ctl->n_fifo;
  const uint32_t n_chunks = (uint32_t)((n + kAdmBlock - 1) / kAdmBlock);
  for (uint32_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const uint64_t k = (uint64_t)c * kAdmBlock + threadIdx.x;
    uint8_t flag = 0;
    if (k < n) {
      const uint32_t i = a.fifo[k];
      if (a.wait[i] != kNotWaiting) {
        const uint32_t bit = 1u << (i & 31);
        if (atomicAnd(&a.sub[i >> 5], ~bit) & bit) {
          atomicAdd(&a.group_sub[i / kGroupRecords], 0xFFFFFFFFu);
          flag = 3;
        } else {
          const uint32_t f = a.c.flags[i];
          const uint32_t kind = f & AM_KIND_MASK;
          const bool can_be_due = kind == AM_KIND_INTERVAL || kind == AM_KIND_CRON_EVERY || kind == AM_KIND_CRON_SPEC;
          if (is_live(f) && can_be_due && !held_run(a.since[i], [&] { return a.c.finished_at[i]; }, [&] { return f; }))
            flag = 1;
          else
            a.wait[i] = kNotWaiting;
        }
      }
      a.cand[k] = flag;
    }
    uint32_t total;
    (void)adm_block_scan(flag ? 1u : 0u, s_warp, &total);
    if (threadIdx.x == 0) a.chunk[c] = total;
  }
}

// One CTA: exclusive prefix of n values in place, returns their sum (the loop of scan_groups_kernel).
__device__ uint32_t adm_scan_in_place(uint32_t* v, uint32_t n, uint32_t* s_warp, uint32_t* s_carry) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) *s_carry = 0;
  __syncthreads();
  for (uint32_t b0 = 0; b0 < n; b0 += blockDim.x) {
    const uint32_t j = b0 + (uint32_t)tid;
    const uint32_t x = j < n ? v[j] : 0u;
    const uint32_t incl = warp_inclusive_scan(x, lane);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const uint32_t t = s_warp[lane];
      s_warp[lane] = warp_inclusive_scan(t, lane) - t;
    }
    __syncthreads();
    const uint32_t excl = *s_carry + s_warp[warp] + incl - x;
    if (j < n) v[j] = excl;
    __syncthreads();
    if (tid == (int)blockDim.x - 1) *s_carry = excl + x;
    __syncthreads();
  }
  const uint32_t total = *s_carry;
  __syncthreads();
  return total;
}

// One CTA of 1024 threads: the ranks' offsets and the cut.
__global__ void __launch_bounds__(1024) adm_plan_kernel(const AdmParams a) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const uint32_t n_chunks = (uint32_t)((a.ctl->n_fifo + kAdmBlock - 1) / kAdmBlock);
  const uint64_t D = adm_scan_in_place(a.chunk, n_chunks, s_warp, &s_carry);
  const uint64_t F = adm_scan_in_place(a.group_sub, a.n_groups, s_warp, &s_carry);
  if (threadIdx.x == 0) {
    const uint64_t B = a.budget;
    const uint64_t adm_def = D < B ? D : B;
    const uint64_t room = B - adm_def;
    const uint64_t adm_fresh = F < room ? F : room;
    AdmCtl* q = a.ctl;
    q->n_def_cand = D;
    q->n_fresh = F;
    q->room = room;
    q->n_keep = D - adm_def;
    q->n_new = F - adm_fresh;
    q->n_candidates = D + F;
    q->n_admitted = adm_def + adm_fresh;
  }
}

// Per FIFO entry: the first `budget` candidates are admitted, the others stay (in order, into `keep`).
__global__ void __launch_bounds__(kAdmBlock) adm_fifo_kernel(const AdmParams a) {
  __shared__ uint32_t s_warp[kAdmBlock / 32];
  const uint64_t n = a.ctl->n_fifo;
  const uint32_t n_chunks = (uint32_t)((n + kAdmBlock - 1) / kAdmBlock);
  for (uint32_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const uint64_t k = (uint64_t)c * kAdmBlock + threadIdx.x;
    const uint8_t flag = k < n ? a.cand[k] : 0;
    uint32_t total;
    const uint64_t rank = a.chunk[c] + adm_block_scan(flag ? 1u : 0u, s_warp, &total);
    if (flag) {
      const uint32_t i = a.fifo[k];
      if (rank < a.budget) {
        a.wait[i] = kNotWaiting;
        if (flag == 1) adm_force(a, i);
      } else {
        a.keep[rank - a.budget] = i;
        if (flag == 3) adm_trim(a, i);
      }
    }
  }
}

// One word per thread, one group per CTA: the fresh candidates ranked by slot; those at or past the room left are
// deferred (trimmed, waiting since T, into `fresh` in slot order).
__global__ void __launch_bounds__(kGroupWords) adm_fresh_kernel(const AdmParams a) {
  __shared__ uint32_t s_warp[kGroupWords / 32];
  if (a.ctl->n_new == 0) return;  // (uniform: every fresh candidate fits)
  const uint64_t room = a.ctl->room;
  const uint32_t g = blockIdx.x, t = threadIdx.x;
  uint32_t m = a.sub[(size_t)g * kGroupWords + t];
  uint32_t total;
  uint64_t rank = a.group_sub[g] + adm_block_scan((uint32_t)__popc(m), s_warp, &total);
  if (a.group_sub[g] + total <= room) return;  // (uniform: the whole group is admitted)
  const uint32_t base = g * kGroupRecords + t * 32u;
  for (; m; m &= m - 1, ++rank) {
    if (rank < room) continue;
    const uint32_t i = base + (uint32_t)(__ffs((int)m) - 1);
    adm_trim(a, i);
    a.wait[i] = a.T;
    a.fresh[rank - room] = i;
  }
}

// Keys of the admission order: (second, slot).
__device__ __forceinline__ bool adm_before(int64_t s, uint32_t i, int64_t t, uint32_t j) {
  return s < t || (s == t && i < j);
}

// The kept entries (ascending by key) and the new ones (all at second T, ascending by slot) merged into the FIFO: every
// element's position is its own index plus the number of the other list's keys below it.  Also the last tick's backlog
// numbers.
__global__ void adm_merge_kernel(const AdmParams a) {
  AdmCtl* q = a.ctl;
  const uint64_t nk = q->n_keep, nn = q->n_new, n = nk + nn;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n; k += stride) {
    uint32_t slot;
    uint64_t pos;
    if (k < nk) {
      slot = a.keep[k];
      const int64_t s = a.wait[slot];
      uint64_t lo = 0, hi = s < a.T ? 0 : nn;  // the new keys below (s, slot)
      if (s == a.T) {
        while (lo < hi) {
          const uint64_t mid = (lo + hi) / 2;
          if (a.fresh[mid] < slot) lo = mid + 1; else hi = mid;
        }
      }
      pos = k + (s == a.T ? lo : hi);
    } else {
      slot = a.fresh[k - nk];
      uint64_t lo = 0, hi = nk;  // the kept keys below (T, slot)
      while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        const uint32_t j = a.keep[mid];
        if (adm_before(a.wait[j], j, a.T, slot)) lo = mid + 1; else hi = mid;
      }
      pos = (k - nk) + lo;
    }
    a.fifo[pos] = slot;
    if (pos == 0) q->oldest = a.wait[slot];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    q->n_fifo = n;
    q->n_deferred = n;
    if (n == 0) q->oldest = INT64_MAX;
  }
}

// am_sweep_next_due: a slot still waiting for admission is due at T + 1 (also the test "does any slot wait" of the
// blocked simulation's refusal).
__global__ void adm_next_due_kernel(const uint32_t* __restrict__ fifo, const int64_t* __restrict__ wait, const AdmCtl* ctl,
                                    int64_t T, unsigned long long* out) {
  const uint64_t n = ctl->n_fifo, stride = (uint64_t)gridDim.x * blockDim.x;
  bool any = false;
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n && !any; k += stride)
    any = wait[fifo[k]] != kNotWaiting;
  if (any) atomicMin(out, biased_key(T + 1));
}

// What am_sweep_deferred reports for slot i: the second since which it waits for admission, kNotWaiting when it does
// not.  The one definition of the value: the dense query and am_sweep_select's mark pass call it.
__device__ __forceinline__ int64_t adm_wait(const int64_t* __restrict__ wait, uint32_t i) { return wait[i]; }

// am_sweep_deferred: adm_wait of the slots first + k (idx == NULL) or first + idx[k], k < n.
__global__ void adm_gather_kernel(const int64_t* __restrict__ wait, uint32_t first, const uint32_t* __restrict__ idx,
                                  uint32_t n, int64_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = adm_wait(wait, first + (idx ? idx[k] : k));
}

// am_sweep_select's mark pass over the slots [first, first + n): one CTA per 8192-slot group of the range (slot
// first + j is in group j / 8192), one slot per thread and step.  Slot first + j matches when its value v — adm_wait
// when `wait` is given (AM_SEL_WAITING), else held_run_start on `since` — is set (not INT64_MIN) and v <= before.  Bit
// j of `bits` is set iff it matches (every word of the CTA's group is written), group_count[g] = the group's matches
// (scan_groups_kernel's input), acc[1] += them and acc[0] = min(acc[0], biased_key(least match)) with one atomic each
// per CTA.  Reads 8 B per slot (since or wait); finishedAt and the flags only where since is set.
__global__ void __launch_bounds__(kGroupWords) select_mark_kernel(DevCols c, const int64_t* __restrict__ since,
                                                                  const int64_t* __restrict__ wait, bool remedy,
                                                                  uint32_t first, uint32_t n, int64_t before,
                                                                  uint32_t* bits, uint32_t* group_count,
                                                                  unsigned long long* acc) {
  __shared__ uint32_t s_cnt[kGroupWords / 32];
  __shared__ unsigned long long s_min[kGroupWords / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t g = blockIdx.x;
  uint32_t cnt = 0;
  unsigned long long best = ~0ull;
#pragma unroll 4
  for (uint32_t r = 0; r < kGroupRecords / kGroupWords; ++r) {  // step r: slots j0 .. j0 + 255, words j0 / 32 + warp
    const uint32_t j0 = g * kGroupRecords + r * kGroupWords;
    const uint32_t j = j0 + threadIdx.x;
    bool m = false;
    if (j < n) {
      const int64_t v = wait ? adm_wait(wait, first + j) : held_run_start(c, since, first + j, remedy);
      m = v != kNotWaiting && v <= before;
      if (m && biased_key(v) < best) best = biased_key(v);
    }
    const uint32_t word = __ballot_sync(kFull, m);
    if (lane == 0) {
      bits[j0 / 32u + warp] = word;
      cnt += (uint32_t)__popc(word);
    }
  }
  best = warp_min(best);
  if (lane == 0) {
    s_cnt[warp] = cnt;
    s_min[warp] = best;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (uint32_t k = 0; k < kGroupWords / 32; ++k) {
      t += s_cnt[k];
      best = s_min[k] < best ? s_min[k] : best;
    }
    group_count[g] = t;
    if (t) {
      atomicAdd(acc + 1, (unsigned long long)t);
      atomicMin(acc, best);
    }
  }
}

}  // namespace amsweep
