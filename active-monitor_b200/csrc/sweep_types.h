// sweep_types.h — constants, kernel parameter blocks and the launch macros shared by the
// tick kernels (sweep_kernels.cuh), the exchange kernels (gather_kernels.cuh) and the host
// runtime (sweep.cu, gather.cu).  No kernel definitions here: both .cu files include it.
#pragma once
#ifndef AMSWEEP_EMULATE  // tests/emu compiles these files for the CPU (cuda_emu.h supplies the model)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/amsweep.h"
#include "civil.h"
#include "tz_eval.h"

// Kernel launches are spelled through two macros so that tests/emu can compile the host
// runtime (sweep.cu) for the CPU emulator as well.  AM_LAUNCH is the plain <<<>>> launch;
// AM_LAUNCH_PDL adds the programmatic-stream-serialization attribute (programmatic dependent
// launch): the kernel may be scheduled while its predecessor in the stream drains and calls
// pdl_wait() (griddepcontrol.wait) before it touches anything the predecessor wrote — the
// launch latency between the four small kernels of a tick disappears behind the sweep's tail.
#ifndef AM_LAUNCH
#ifndef AMSWEEP_EMULATE
#define AM_LAUNCH(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#define AM_LAUNCH_PDL(kernel, grid, block, strm_, ...)                                    \
  do {                                                                                    \
    cudaLaunchConfig_t _cfg = {};                                                         \
    _cfg.gridDim = dim3(grid);                                                            \
    _cfg.blockDim = dim3(block);                                                          \
    _cfg.stream = (strm_);                                                                \
    cudaLaunchAttribute _at[1];                                                           \
    _at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                       \
    _at[0].val.programmaticStreamSerializationAllowed = 1;                                \
    _cfg.attrs = _at;                                                                     \
    _cfg.numAttrs = 1;                                                                    \
    (void)cudaLaunchKernelEx(&_cfg, kernel, __VA_ARGS__);                                 \
  } while (0)
#else
#define AM_LAUNCH(kernel, grid, block, stream, ...) ((void)(stream), emu::launch(kernel, dim3(grid), dim3(block), __VA_ARGS__))
#define AM_LAUNCH_PDL(kernel, grid, block, stream, ...) ((void)(stream), emu::launch(kernel, dim3(grid), dim3(block), __VA_ARGS__))
#endif
#endif

namespace amsweep {

#ifndef AM_BLOCK
#define AM_BLOCK 256
#endif
constexpr int kBlock = AM_BLOCK;
constexpr int kWarps = kBlock / 32;
constexpr int kRecPerWarp = 128;             // 2 halves x 32 lanes x 2 records
constexpr int kTile = kWarps * kRecPerWarp;  // 1024 records per CTA
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kNumAcc = 16;  // == number of u64 fields of am_tick_stats_t
constexpr int kMaxWorld = 16;

// A "group" is the unit of the list rebuild: 8 tiles = 8192 records = 256 bitmap words = one
// expand CTA with one word per thread.
constexpr int kGroupTiles = 8;
constexpr uint32_t kGroupRecords = kGroupTiles * kTile;  // 8192
constexpr uint32_t kGroupWords = kGroupRecords / 32;     // 256
constexpr uint32_t kTileWords = kTile / 32;              // 32
static_assert(kBlock == 256 && kTile == 1024, "bitmap layout: 32 words per tile, 4 per warp");

struct DevCols {
  uint64_t *minute, *hour, *dom, *month, *dow;
  int32_t* ras;
  uint32_t* flags;
  int64_t* finished_at;
  int32_t *runs_limit, *reset_interval;
  int32_t *success, *failed, *remedy_success, *remedy_failed, *remedy_total;
  int64_t* remedy_finished_at;
};

// The cron masks as the on-minute sweep reads them: one bit plane per value a field of the tick's
// one-hot words can take (minute 0..59, hour 0..23, dom 1..31, month 1..12, dow 0..6) plus the robfig
// star bit (bit 63 of dom OR bit 63 of dow), each a bitmap over the shard with one bit per record.
// Bit r of plane P is bit v of the field's mask of record r, set only for CRON_SPEC records that are
// not bound to a time zone (flags bits 24..31 zero); every other record is zero in every plane.  A
// mask bit outside those ranges is never tested by cron_matches, so it has no plane.  Plane-major:
// plane P is words [P * words, (P + 1) * words).  A "segment" is the kRecPerWarp records one warp of
// sweep_tick_kernel owns (4 words of a plane); every write of the canonical masks or of the kind or
// zone bits rebuilds the segments it touched (build_segment_planes); nothing else reads the planes.
// Plane of value v of a field: kPlane<field> + v.
constexpr int kPlaneMinute = 0;   // minute 0..59: planes 0..59
constexpr int kPlaneHour = 60;    // hour 0..23: planes 60..83
constexpr int kPlaneDom = 83;     // dom 1..31: planes 84..114
constexpr int kPlaneMonth = 114;  // month 1..12: planes 115..126
constexpr int kPlaneDow = 127;    // dow 0..6: planes 127..133
constexpr int kPlaneStar = 134;
constexpr int kPlanes = 135;
struct MaskPlanes {
  uint32_t* w;     // [kPlanes * words]
  uint64_t words;  // per plane: cap_padded / 32
};
// The six planes one tick tests (T's UTC minute, hour, dom, month, dow, and the star plane)
struct TickPlanes {
  const uint32_t *minute, *hour, *dom, *month, *dow, *star;
};

// What one tick of one shard leaves behind for the list rebuild (expand_kernel) and for the
// NVLink exchange: the same four arrays whether they are the sweep's own buffers or the copy
// a peer pushed into this GPU's exchange block.
struct TickOut {
  uint32_t* bitmap;        // [n_groups * 256] bit b of word w = record 32 w + b of the shard is emitted
  uint32_t* group_count;   // [n_groups] emitted records per group (REDs of the tiles; zero on entry)
  uint32_t* group_prefix;  // [n_groups + 1] exclusive prefix of group_count (scan_groups_kernel)
  uint32_t* tile_exc;      // [n_tiles] exceptions per tile
  uint32_t* exc_seg;       // [n_tiles * 1024] per tile: exception entries (exc_entry), ascending
};
// An exception entry: the record's offset in its tile above its 8 action bits (a tile's entries ascend by record).
AM_HD uint32_t exc_entry(uint32_t off, uint32_t act) { return (off << 8) | act; }
AM_HD uint32_t exc_offset(uint32_t e) { return e >> 8; }
AM_HD uint32_t exc_action(uint32_t e) { return e & 0xFFu; }

struct SweepParams {
  DevCols c;
  TickPlanes pl;  // read by the MASKS variants instead of the five canonical mask columns
  uint64_t n_records;
  uint64_t shard_base;
  uint64_t seed;
  int64_t T;
  TickWords words;  // T's UTC fields as one-hot words, computed once per tick by the launcher
  uint32_t n_tiles;
  uint32_t mode;
  TickOut out;
  unsigned long long* acc;   // [kNumAcc] statistics accumulators (zero on entry)
  const TickWords* tz_table; // [zones + 1] T's LOCAL fields per registered time zone (entry 0 = UTC), written by
                             // tz_words_kernel ahead of the sweep; NULL when no zone is registered.
                             // WINDOW variant: [256 * kWindowBoxes] the catch-up window's calendar boxes per zone
                             // (civil.h, window_boxes), the unused ones with sec0 = 0
  int64_t* since;            // HOLD variants: [cap] the second of the tick that submitted the slot's running health-check
                             // workflow, kNotInFlight when none (am_sweep_set_hold_in_flight); NULL otherwise
  // TIMEOUT variants (workflow timeouts, am_record_t.wf_timeout): NULL otherwise
  const int32_t* wf_timeout;           // [cap] the slot's workflow timeout in seconds, 0 = none (the latest upsert's)
  int64_t* deadline;                   // [cap] the running workflow's deadline, kNoDeadline when none
  unsigned long long* seg_deadline;    // [cap / kRecPerWarp] per warp segment a lower bound of its deadlines (biased key)
  // DUE variants (open loop, no window, no hold): the due words (due_word, sweep_kernels.cuh) instead of ras and
  // finishedAt, and T - E of the handle's epoch E; NULL / 0 otherwise
  uint32_t* due;
  uint32_t due_t;
  int64_t due_epoch;
};
constexpr int64_t kNotInFlight = INT64_MIN;
constexpr int64_t kNoDeadline = INT64_MAX;
// Remedy hold (am_sweep_set_hold_remedy): a running remedy workflow started at T is kept in the slot's since word as
// T + kRemedyRun.  Every tick second is |T| < 2^55, so a since word >= kRemedyRun / 2 is a remedy run and anything
// below is a health-check run; a check has at most one run of either kind in flight, so they share the word (and the
// deadline word).
constexpr int64_t kRemedyRun = 1ll << 60;
AM_HD bool is_remedy_run(int64_t since) { return since >= kRemedyRun / 2; }
// the start of the run a since word holds, of either kind (kNotInFlight stays kNotInFlight)
AM_HD int64_t run_start(int64_t since) { return is_remedy_run(since) ? since - kRemedyRun : since; }
// a signed second as an unsigned key of the same order (the atomicMin idiom of next_due_kernel); kNoDeadline -> ~0
__device__ __forceinline__ unsigned long long biased_key(int64_t t) { return (unsigned long long)t ^ (1ull << 63); }

struct ScanParams {
  uint32_t* group_count;        // this tick's per-group sums; zeroed again once read
  uint32_t* group_prefix;       // [n_groups + 1]
  unsigned long long* acc;      // acc[1] = n_emitted
  uint32_t* out_count;          // may be NULL: min(n_emitted, cap) for device-side consumers
  uint32_t n_groups, cap;
};

struct ExpandSrc {
  const uint32_t* bitmap;
  const uint32_t* group_prefix;
  const uint32_t* tile_exc;
  const uint32_t* exc_seg;
  uint64_t base;  // added to the shard-local record number to form the output index
  uint32_t n_groups, n_tiles;
};
struct ExpandParams {
  ExpandSrc src[kMaxWorld];  // rank order; the output is their concatenation
  void* out_idx;             // [cap] u32 or u64
  uint8_t* out_act;          // [cap]
  unsigned long long* acc;   // action-bit counts and index checksums of rank `stats_rank` (may be NULL)
  uint64_t stats_base;       // global index of that rank's record 0 (checksums are over global indices)
  uint64_t cap;
  int world, stats_rank, idx_bytes;
};

}  // namespace amsweep
