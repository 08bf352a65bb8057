// host_loops.cpp — the two per-entry host loops of the e2e path, written so that the
// compiler vectorises them (plain strided loops, no tables, no branches) and cloned for
// AVX2 with run-time dispatch: at a few hundred thousand posted results and emitted
// entries per one-second tick they were, with the staging copies, most of the round-1
// e2e step.
//
//   stage_results  am_sweep_post_result: (u64 slot, u8 phase, u8 remedy phase) -> staged
//                  ops (one 64-bit word each) in pinned memory (hcc.go:635/:662/:821/:836 observations)
//   widen_list     am_sweep_tick: (u32 local index, u8 action) -> the caller's
//                  (u64 global index, u32 action) arrays (SURVEY 8b signature)
#include <stddef.h>
#include <stdint.h>

#include "../../include/amsweep.h"

#if defined(__x86_64__) && defined(__GNUC__) && !defined(__clang__) && !defined(AMSWEEP_EMULATE)
#define AM_SIMD_CLONES __attribute__((target_clones("avx2", "default")))
#else
#define AM_SIMD_CLONES
#endif

namespace amsweep_host {

// A staged op is one 64-bit word: slot in the low half, arg (kind | payload) in the high half — one
// stream of stores here, one copy to the device, one 8-B load per op in the kernels.
// returns bit 0: a slot >= capacity, bit 1: a phase outside {0, 1, 2}
AM_SIMD_CLONES
unsigned stage_results(uint64_t n, const uint64_t* __restrict__ idx, const uint8_t* __restrict__ phase,
                       const uint8_t* __restrict__ remedy, uint64_t capacity, uint32_t op_result_kind,
                       uint64_t* __restrict__ ops) {
  uint64_t bad_range = 0;
  uint32_t bad_phase = 0;
  if (remedy) {
    for (uint64_t k = 0; k < n; ++k) {
      const uint64_t i = idx[k];
      const uint32_t p = phase[k], r = remedy[k];
      bad_range |= (uint64_t)(i >= capacity);
      bad_phase |= (uint32_t)(p > AM_PHASE_FAILED) | (uint32_t)(r > AM_PHASE_FAILED);
      const uint32_t bits = (p == AM_PHASE_SUCCEEDED ? AM_F_PENDING_OK : 0u) | (p == AM_PHASE_FAILED ? AM_F_PENDING_FAIL : 0u) |
                            (r != AM_PHASE_NONE ? AM_F_REMEDY_PENDING : 0u) |
                            (r == AM_PHASE_SUCCEEDED ? AM_F_REMEDY_OUTCOME_OK : 0u);
      ops[k] = (uint64_t)(uint32_t)i | ((uint64_t)(op_result_kind | bits) << 32);
    }
  } else {
    for (uint64_t k = 0; k < n; ++k) {
      const uint64_t i = idx[k];
      const uint32_t p = phase[k];
      bad_range |= (uint64_t)(i >= capacity);
      bad_phase |= (uint32_t)(p > AM_PHASE_FAILED);
      const uint32_t bits = (p == AM_PHASE_SUCCEEDED ? AM_F_PENDING_OK : 0u) | (p == AM_PHASE_FAILED ? AM_F_PENDING_FAIL : 0u);
      ops[k] = (uint64_t)(uint32_t)i | ((uint64_t)(op_result_kind | bits) << 32);
    }
  }
  return (bad_range ? 1u : 0u) | (bad_phase ? 2u : 0u);
}

AM_SIMD_CLONES
void widen_list(uint64_t n, uint64_t base, const uint32_t* __restrict__ idx32, const uint8_t* __restrict__ act8,
                uint64_t* __restrict__ idx64, uint32_t* __restrict__ act32) {
  for (uint64_t k = 0; k < n; ++k) idx64[k] = base + idx32[k];
  for (uint64_t k = 0; k < n; ++k) act32[k] = act8[k];
}

// slots of an upsert / remove batch: range check + narrowing; arg = arg0 + k * arg_step (an upsert's record index)
AM_SIMD_CLONES
unsigned stage_slots(uint64_t n, const uint64_t* __restrict__ idx, uint64_t capacity, uint32_t arg0, uint32_t arg_step,
                     uint64_t* __restrict__ ops) {
  uint64_t bad = 0;
  for (uint64_t k = 0; k < n; ++k) {
    bad |= (uint64_t)(idx[k] >= capacity);
    ops[k] = (uint64_t)(uint32_t)idx[k] | ((uint64_t)(arg0 + (uint32_t)k * arg_step) << 32);
  }
  return bad ? 1u : 0u;
}

// flags words `stride` u32 apart (a column, or the flags of packed records): 1 when a 5-field schedule names a
// zone id above `n_zones` — ids are process-local, and only registered ones have offsets on the device
AM_SIMD_CLONES
unsigned unknown_zones(uint64_t n, const uint32_t* __restrict__ flags, uint64_t stride, uint32_t n_zones) {
  uint32_t bad = 0;
  for (uint64_t k = 0; k < n; ++k) {
    const uint32_t f = flags[k * stride];
    bad |= (uint32_t)((f & AM_KIND_MASK) == AM_KIND_CRON_SPEC) & (uint32_t)((f >> AM_F_TZ_SHIFT) > n_zones);
  }
  return bad;
}

}  // namespace amsweep_host
