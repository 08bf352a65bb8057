// sweep.cu — the am_sweep handle and the C-ABI entry points of libamsweep.
//
// Owns one shard of the HealthCheck record array in HBM (16 SoA columns,
// SURVEY.md Appendix B.1) on one CUDA device, the staging area for
// upsert / remove / post_result calls coming from the controller's goroutines
// (hcc.go:170-188 Reconcile workers, hcc.go:635/:662/:821/:836 watch loops),
// and the launch of the tick's kernels (sweep_kernels.cuh) that replace the
// per-CR schedule ladder and remedy state machine for every record at once.
//
// Shape of the host side (round 2):
//   * staged events are 64-bit words (slot, arg) (+ 96-B records for upserts) in pinned
//     memory, double-buffered: a tick swaps the buffers under the staging lock and
//     releases it at once — callers never wait for a copy or a kernel;
//   * posted events are copied to the device in chunks WHILE they are being posted (copy
//     stream), so at tick time only the tail is left;
//   * the list rebuild writes (u32 local index, u8 action) straight into mapped pinned
//     host memory and the statistics into a mapped struct: ONE stream synchronisation per
//     tick, no device-to-host copy call, and am_sweep_tick_view hands that memory to the
//     caller without another pass;
//   * every device operation of a handle is ordered after the previous one even when they
//     are issued on different streams (am_sweep_tick_device takes the caller's stream);
//   * am_sweep_tick, _tick_view, _tick_device and _tick_shard run one path (run_tick): the
//     refusals, the drain, the sweep and the commit of the previous tick's second; the sweep
//     variant comes from one table (sweep_variant);
//   * am_sweep_run_ticks and am_sweep_simulate run one path for runs of ticks (begin_run, run_rows, run_blocks) around
//     their own tick loops;
//   * fixed-size device arrays, pinned host arrays, events and streams are recorded on the handle as they are made
//     (dev_array, host_array, new_event, new_stream): am_sweep_destroy frees that list;
//   * every kernel is launched through launch / launch_pdl, which count it and return its launch error.
//
// There is deliberately no CPU path in this file: without a CUDA device
// am_sweep_create fails with AM_E_DEVICE.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "admission_kernels.cuh"
#include "checkpoint_kernels.cuh"
#include "checkpoint_pack_kernels.cuh"
#include "sweep_internal.h"
#include "sweep_kernels.cuh"
#include "tz.h"

using namespace amsweep;

namespace amsweep_host {
unsigned stage_results(uint64_t n, const uint64_t* idx, const uint8_t* phase, const uint8_t* remedy, uint64_t capacity,
                       uint32_t op_result_kind, uint64_t* ops);
void widen_list(uint64_t n, uint64_t base, const uint32_t* idx32, const uint8_t* act8, uint64_t* idx64, uint32_t* act32);
unsigned stage_slots(uint64_t n, const uint64_t* idx, uint64_t capacity, uint32_t arg0, uint32_t arg_step, uint64_t* ops);
unsigned unknown_zones(uint64_t n, const uint32_t* flags, uint64_t stride, uint32_t n_zones);
}  // namespace amsweep_host

namespace {
// Reason of the last failed am_sweep_create, process-wide: a cgo caller may be moved to
// another OS thread between the failing call and am_last_error_detail(NULL).
std::mutex g_create_mu;
std::string g_create_error;
void set_create_error(const std::string& s) {
  std::lock_guard<std::mutex> lk(g_create_mu);
  g_create_error = s;
}

// A growable array in pinned host memory or in device memory; its contents do not survive growth.
template <bool kPinned>
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes, unsigned flags = cudaHostAllocDefault) {
    if (bytes <= cap) return cudaSuccess;
    release();
    size_t want = bytes + bytes / 2 + 4096;
    cudaError_t e = kPinned ? cudaHostAlloc(&p, want, flags) : cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) (void)(kPinned ? cudaFreeHost(p) : cudaFree(p)); p = nullptr; cap = 0; }
};
using PinnedBuf = Buf<true>;
using DevBuf = Buf<false>;

// A small table uploaded from the host on the tick's stream.  The device array and the pinned copy are allocated
// at their full size, the device one zeroed, at the first upload.
struct Upload {
  void* dev = nullptr;
  void* pin = nullptr;
  cudaEvent_t copied = nullptr;  // the last upload has left `pin`
  bool pending = false;
};

// What am_sweep_destroy frees: every fixed-size allocation, event and stream of a handle, recorded as it is made.
struct Owned {
  enum Kind { kDevice, kPinned, kEvent, kStream } kind;
  void* p;
};

// One of the two staging areas for controller events.  The pinned arrays are appended to
// under am_sweep::mu; the device twins receive them in chunks on the copy stream.
struct Staging {
  PinnedBuf ops, recs;   // an op = one 64-bit word: slot | arg << 32
  DevBuf d_ops, d_recs;
  // the first op index of every post call, ascending (reservation order), and its device copy: a drain of more ops than
  // a call tag spans tells two post calls apart by it (capture_superseded_kernel)
  std::vector<uint32_t> calls;
  DevBuf d_calls;
  size_t n_ops = 0, n_recs = 0;
  size_t flushed_ops = 0, flushed_recs = 0;  // already enqueued for copy to the device twins
  uint32_t n_state = 0, n_result = 0, n_spec = 0;
  bool any_wf = false;  // an upsert or spec update staged here carries a non-zero wf_timeout
  // am_sweep_post_result calls that have reserved a range of the op arrays and are filling it
  // OUTSIDE the lock (the controller's workers post concurrently, hcc.go:170-188): while there are
  // any, the arrays may not move, nothing past `flushed_ops` is known complete, and the drain waits
  int writers = 0;
  size_t done_ops = 0;  // every op below this index is staged completely (== n_ops when writers == 0)
  std::vector<std::pair<size_t, size_t>> done_ranges;  // completed ranges above the prefix (other writers still below them)
  uint64_t hwm = 0;                          // highest upserted slot + 1
  cudaEvent_t copied = nullptr;              // the last copy out of the pinned arrays
  bool copy_pending = false;
  cudaEvent_t drained = nullptr;             // the last kernel that read the device twins
  bool drain_pending = false;
};

// One of the two buffer sets a tick writes (by tick parity): a consumer of tick k — the
// list rebuild, or the NVLink exchange on another stream — overlaps the sweep of tick k+1.
struct TickSet {
  TickOut out{};
  unsigned long long* acc = nullptr;
  cudaEvent_t consumed = nullptr;
  bool consumed_pending = false;
  // an am_sweep_tick_shard left its statistics in `acc` and no exchange has published (and so re-armed) them yet:
  // the next tick on this set starts from zero
  bool unpublished = false;
};

// A delta chain's range on the handle that applied its last link (am_sweep_restore_delta): that link's checksum and the
// handle's tick count when it was applied.
struct CkptLink {
  uint64_t first_global, n, checksum, ticks;
};

constexpr size_t kFlushOps = 32768;   // staged ops per early host-to-device chunk
constexpr size_t kFlushRecs = 8192;   // staged upsert records per early chunk
}  // namespace

struct am_sweep {
  int device = 0;
  int sms = 1;  // multiprocessors of `device`: grid size of the grid-stride kernels
  uint64_t capacity = 0, cap_padded = 0, shard_base = 0;
  uint64_t n_records = 0;  // high-water mark
  DevCols cols{};
  MaskPlanes planes{};             // the on-minute sweep's copy of the mask columns as bit planes
  uint32_t* seg_dirty = nullptr;   // [cap_padded / kRecPerWarp] segments a drain's state ops touched
  TickSet set[2];
  uint32_t parity = 0;
  int last_shard_parity = -1;
  uint32_t* due_idx[2] = {nullptr, nullptr};   // HBM list ring (streaming mode)
  uint8_t* due_action[2] = {nullptr, nullptr};
  // host-visible list of the last host tick: mapped pinned memory written by expand_kernel
  PinnedBuf host_out;
  uint64_t host_out_entries = 0;  // capacity in entries
  uint64_t host_n = 0;            // entries of the last host tick
  am_tick_stats_t* h_stats = nullptr;  // pinned + mapped
  am_tick_stats_t* d_stats_mapped = nullptr;
  cudaStream_t stream = nullptr;   // the handle's own stream
  cudaStream_t cstream = nullptr;  // staging copies
  cudaStream_t last_stream = nullptr;  // where the handle's last device operation was issued
  bool has_last = false;
  cudaEvent_t ev_last = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t evp[3] = {nullptr, nullptr, nullptr};  // profiling: before sweep, after sweep, after publish
  bool profiling = false, profiled = false;
  std::mutex mu;  // guards the staging areas
  std::condition_variable cv;  // a staging area's `writers` dropped to zero
  std::atomic_flag ticking = ATOMIC_FLAG_INIT;
  Staging stage[2];
  int cur = 0;                // the staging area callers append to
  uint32_t* marks = nullptr;  // [3 * cap_padded] per-slot {latest state op, latest phase, latest remedy phase}
  uint32_t* spec_marks = nullptr;  // [cap_padded] per-slot latest spec update, allocated by the first drain that has one
  PinnedBuf pin_in;
  DevBuf dev_in;
  // named time zones: one UTC offset per registered zone (tz.h) on the device, refreshed when the
  // registry grows or a tick leaves the window [tz_lo, tz_hi) in which no zone changes its offset
  uint64_t tz_version = ~0ull;
  uint32_t tz_n = 0;  // zones + 1; 0 or 1 = nothing registered
  int64_t tz_lo = 0, tz_hi = 0;
  bool tz_aligned = true;  // every offset a whole number of minutes
  Upload tz_off;                 // [kMaxZones + 1] int32
  TickWords* tz_table = nullptr;  // [kMaxZones + 1], written by tz_words_kernel
  // catch-up ticks (AM_SWEEP_CATCH_UP): the second of the previous tick, and the device table of a window's
  // calendar boxes ([kMaxZones + 1][kWindowBoxes], allocated at the first catch-up tick that needs it)
  bool has_prev = false;
  int64_t prev_T = 0;
  Upload win_boxes;
  // hold in flight (am_sweep_set_hold_in_flight): per slot the second of the tick that submitted its running health-check
  // workflow, kNotInFlight when none ([cap_padded], allocated when the hold is first turned on)
  bool hold = false;
  int64_t* since = nullptr;
  // remedy hold (am_sweep_set_hold_remedy, only with the hold): a running remedy workflow is kept in the same since and
  // deadline words, its since as T + kRemedyRun
  bool remedy = false;
  // workflow timeouts (am_record_t.wf_timeout), allocated by the first drain that stages a non-zero one: per slot the
  // latest upsert's timeout and the running workflow's deadline, per warp segment a lower bound of its deadlines, and
  // the tick's timed-out list (room for every slot)
  int32_t* wf_timeout = nullptr;
  int64_t* deadline = nullptr;
  unsigned long long* seg_deadline = nullptr;
  uint32_t* to_idx = nullptr;
  int64_t* to_since = nullptr;
  uint32_t* to_count = nullptr;
  bool to_ran = false;      // the last tick ran expire_runs_kernel: its list is on the device
  bool to_fetched = false;  // ... and has been copied to to_host / rto_host, sorted
  std::vector<std::pair<uint32_t, int64_t>> to_host;   // health-check runs: (slot, since)
  std::vector<std::pair<uint32_t, int64_t>> rto_host;  // remedy runs: (slot, start)
  // simulated workflows (am_sweep_simulate), allocated at the first call: per warp segment a lower bound of its held
  // runs' simulated ends (biased key), for the tick-by-tick completion pass
  unsigned long long* sim_end = nullptr;
  // status changes (am_sweep_set_track_changes), allocated at the first enable: one bit per slot that the coming tick
  // changes ([n_groups * kGroupWords], drains and the tick add to it, the list kernel clears it), the last tick's
  // ascending slot list ([cap_padded]), and the per-group counts, offsets and total of the compaction
  bool track = false;
  uint32_t* chg_bits = nullptr;
  uint32_t* chg_list = nullptr;
  uint32_t* chg_group = nullptr;
  uint32_t* chg_prefix = nullptr;
  unsigned long long* chg_acc = nullptr;  // scan_groups_kernel's accumulators: [1] = entries in chg_list
  bool chg_listed = false;   // the last tick built its list on the device
  bool chg_fetched = false;  // ... and its length has been read into chg_n
  uint64_t chg_n = 0;
  // change details (am_sweep_set_change_details, only with tracking), allocated at the first enable: per slot the
  // AM_CHG_* bits and the run start a pass captured ([cap_padded] each, meaningful while the slot's bit is set), the
  // same of the last tick's list by entry, and the tick the list belongs to (its buffer set, second and closed-loop
  // mode) for the action bytes
  bool details = false;
  uint8_t* det_applied = nullptr;
  int64_t* det_start = nullptr;
  uint8_t* det_e_applied = nullptr;  // ... and the pairs of the last tick's list, by entry ([cap_padded] each)
  int64_t* det_e_start = nullptr;
  int chg_parity = 0;
  int64_t chg_T = 0;
  bool chg_closed = false;
  bool det_listed = false;  // the last list was built with details on (a list from before they were on has none)
  std::string last_error;
  std::atomic<uint64_t> launches{0};  // (a restore launches outside the tick guard)
  double last_ms = -1.0;
  uint64_t seed = 0;
  bool early_results = true;  // AMSWEEP_EARLY_RESULTS=0: every posted result is applied inside the sweep
  Staging* pend_clear = nullptr;  // a host tick's drain leaves clear_marks_kernel for after the tick's kernels
  size_t pend_clear_n = 0;
  bool pend_clear_spec = false;   // ... and that drain had spec updates
  std::vector<Owned> owned;
  std::mutex owned_mu;  // guards appends to `owned` (a restore allocates outside the tick guard)
  // checkpoints (am_sweep_checkpoint / am_sweep_restore), allocated at the first one and serialised by ck_mu (they share
  // it all): the blob's sections in HBM (room for every section of every slot of capacity), the pass's checksum sum and
  // zone marks (device and pinned), the stream that copies blobs to and from the caller while ticks go on, and two
  // pinned chunks that a restore's upload alternates between.
  std::mutex ck_mu;
  char* ck_dev = nullptr;
  unsigned long long* ck_meta = nullptr;    // [0] checksum sum, then 8 words of zone marks
  unsigned long long* ck_meta_h = nullptr;  // pinned copy
  cudaStream_t ck_stream = nullptr;
  cudaEvent_t ck_ev = nullptr;  // the pass is done (and its meta copied)
  char* ck_pin[2] = {nullptr, nullptr};
  cudaEvent_t ck_pin_ev[2] = {nullptr, nullptr};
  bool ck_pin_pending[2] = {false, false};
  // delta chains (am_sweep_checkpoint_chain / _delta / am_sweep_restore_delta), also under ck_mu.  On a producer,
  // allocated when its first chain starts: the previous link's sections over the chain's range (the root's layout; room
  // for a full blob of capacity), the diff's bitmap ([groups of capacity * kGroupWords]) and per-group counts and
  // offsets.  On both sides, at the first chain or delta restore: a delta's slot offsets ([cap_padded]) and the
  // scan's accumulators ([1] the changed slots, [2] a bad offset), device and pinned.
  char* ckd_base = nullptr;
  uint32_t* ckd_bits = nullptr;
  uint32_t* ckd_group = nullptr;
  uint32_t* ckd_prefix = nullptr;
  uint32_t* ckd_off = nullptr;
  unsigned long long* ckd_acc = nullptr;
  unsigned long long* ckd_acc_h = nullptr;
  // packed checkpoints (am_sweep_set_checkpoint_packing), also under ck_mu: whether producers pack, and, at the first
  // packed checkpoint or restore, the packed staging area (a directory and payload as large as a delta with every slot
  // of capacity changed and every section), the encode's per-block sizes, their scan and base values, and the
  // accumulators ([1] the payload's words, [2] a refused directory or block), device and pinned.
  bool ck_packing = false;
  char* ckp_dev = nullptr;
  uint32_t* ckp_words = nullptr;
  uint32_t* ckp_prefix = nullptr;
  int64_t* ckp_base = nullptr;
  unsigned long long* ckp_acc = nullptr;
  unsigned long long* ckp_acc_h = nullptr;
  // the producer's chain: its range, the root's switches, the last link's checksum, sequence number and P
  bool chain = false;
  uint64_t chain_first = 0, chain_n = 0, chain_checksum = 0, chain_seq = 0;
  uint32_t chain_switches = 0;
  int64_t chain_prev_tick = 0;
  // the restorer's chains: per range the last link it applied (a full restore starts an entry), and the ticks run by
  // any entry point (a delta applies only to a handle that has not ticked since its parent)
  std::vector<CkptLink> links;
  uint64_t ticks = 0;
  // submit budget (am_sweep_set_submit_budget, only with the hold): the most SUBMIT_HC entries a tick emits, and the
  // admission state, allocated at the first finite budget (admission_kernels.cuh): per slot the second since which it
  // waits, the FIFO of waiting slots and this tick's kept and new ones, a byte per FIFO entry, one bit per slot of
  // fresh submissions, the per-group and per-chunk counts and the counters
  uint64_t budget = UINT64_MAX;
  int64_t* adm_wait = nullptr;
  uint32_t* adm_fifo = nullptr;
  uint32_t* adm_keep = nullptr;
  uint32_t* adm_fresh = nullptr;
  uint8_t* adm_cand = nullptr;
  uint32_t* adm_sub = nullptr;
  uint32_t* adm_group_sub = nullptr;
  uint32_t* adm_chunk = nullptr;
  AdmCtl* adm_ctl = nullptr;
  // sparse state queries (am_sweep_select), allocated at the first call that reaches the device: the mark pass's bitmap
  // ([groups of capacity * kGroupWords]), per-group counts and offsets, the matches' slots relative to the call's first
  // ([cap_padded]) and the accumulators ([0] the least match as a biased key, [1] the matches)
  uint32_t* sel_bits = nullptr;
  uint32_t* sel_group = nullptr;
  uint32_t* sel_prefix = nullptr;
  uint32_t* sel_list = nullptr;
  unsigned long long* sel_acc = nullptr;
  // due words (due_word, sweep_kernels.cuh) of the open-loop plain ticks, allocated at the first one ([cap_padded]): exact
  // for slots [0, due_end) against the epoch due_epoch while due_valid.  The few writers of ras and finishedAt the common
  // flows run keep them (the DUE sweep variants, the drain's upserts, spec updates and results, delta restores); every
  // other one clears due_valid, and the next such tick rebuilds them (due_tick).  A caller handed ras or finishedAt by
  // am_sweep_column_ptr may write them unseen: due_exposed, never cleared, keeps the handle on the variants that read
  // both columns.
  uint32_t* due = nullptr;
  int64_t due_epoch = 0;
  uint64_t due_end = 0;
  bool due_valid = false;
  std::atomic<bool> due_exposed{false};
};

namespace {

#define AM_CUDA(h, expr)                                                              \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      char _b[512];                                                                   \
      snprintf(_b, sizeof _b, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      if (h) (h)->last_error = _b; else set_create_error(_b);                         \
      return _e == cudaErrorMemoryAllocation ? AM_E_NOMEM : AM_E_DEVICE;              \
    }                                                                                 \
  } while (0)

// Every kernel launch of the handle: counted for am_sweep_launch_count, and its launch error returned (for AM_CUDA).
template <class... P, class... A>
cudaError_t launch(am_sweep* h, void (*k)(P...), dim3 grid, dim3 block, cudaStream_t s, const A&... args) {
  AM_LAUNCH(k, grid, block, s, args...);
  h->launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}
// ... with programmatic dependent launch (AM_LAUNCH_PDL)
template <class... P, class... A>
cudaError_t launch_pdl(am_sweep* h, void (*k)(P...), dim3 grid, dim3 block, cudaStream_t s, const A&... args) {
  AM_LAUNCH_PDL(k, grid, block, s, args...);
  h->launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

constexpr size_t kColElem[16] = {8, 8, 8, 8, 8, 4, 4, 8, 4, 4, 4, 4, 4, 4, 4, 8};

void** col_slot(DevCols& c, int k) {
  void** slots[16] = {(void**)&c.minute,         (void**)&c.hour,          (void**)&c.dom,
                      (void**)&c.month,          (void**)&c.dow,           (void**)&c.ras,
                      (void**)&c.flags,          (void**)&c.finished_at,   (void**)&c.runs_limit,
                      (void**)&c.reset_interval, (void**)&c.success,       (void**)&c.failed,
                      (void**)&c.remedy_success, (void**)&c.remedy_failed, (void**)&c.remedy_total,
                      (void**)&c.remedy_finished_at};
  return slots[k];
}
void* const* cols_member(const am_record_cols_t* c, int k) {
  void* const* slots[16] = {(void* const*)&c->minute,         (void* const*)&c->hour,
                            (void* const*)&c->dom,            (void* const*)&c->month,
                            (void* const*)&c->dow,            (void* const*)&c->ras,
                            (void* const*)&c->flags,          (void* const*)&c->finished_at,
                            (void* const*)&c->runs_limit,     (void* const*)&c->reset_interval,
                            (void* const*)&c->success,        (void* const*)&c->failed,
                            (void* const*)&c->remedy_success, (void* const*)&c->remedy_failed,
                            (void* const*)&c->remedy_total,   (void* const*)&c->remedy_finished_at};
  return slots[k];
}

// The high-water mark moves under the tick guard; am_sweep_size reads it from any thread without taking the guard.
void set_hwm(am_sweep* h, uint64_t v) { __atomic_store_n(&h->n_records, v, __ATOMIC_RELAXED); }

struct TickGuard {
  am_sweep* h;
  bool ok;
  explicit TickGuard(am_sweep* hh) : h(hh), ok(!hh->ticking.test_and_set(std::memory_order_acquire)) {}
  ~TickGuard() { if (ok) h->ticking.clear(std::memory_order_release); }
};

// Every device operation of a handle is ordered after the previous one.  They normally
// share a stream; when the stream changes (am_sweep_tick_device on a caller stream, then a
// read on the handle's own, ...) the new stream waits for an event recorded on the old one.  wait_last only makes
// `s` wait; order_on also makes `s` the stream of the handle's last operation.
int wait_last(am_sweep* h, cudaStream_t s) {
  if (h->has_last && h->last_stream != s) {
    AM_CUDA(h, cudaEventRecord(h->ev_last, h->last_stream));
    AM_CUDA(h, cudaStreamWaitEvent(s, h->ev_last, 0));
  }
  return AM_OK;
}
int order_on(am_sweep* h, cudaStream_t s) {
  if (int rc = wait_last(h, s)) return rc;
  h->last_stream = s;
  h->has_last = true;
  return AM_OK;
}

// The first half of every call's device work: the handle's device current and `s` ordered after its last operation.
int set_stream(am_sweep* h, cudaStream_t s) {
  AM_CUDA(h, cudaSetDevice(h->device));
  return order_on(h, s);
}

void own(am_sweep* h, Owned::Kind kind, void* p) {
  std::lock_guard<std::mutex> lk(h->owned_mu);
  h->owned.push_back({kind, p});
}

// A fixed-size device array owned by the handle until am_sweep_destroy; zeroed on `s` when `zero`.
template <class T>
cudaError_t dev_array(am_sweep* h, T** p, size_t bytes, cudaStream_t s, bool zero = true) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, bytes);
  if (e != cudaSuccess) return e;
  own(h, Owned::kDevice, q);
  *p = (T*)q;
  return zero ? cudaMemsetAsync(q, 0, bytes, s) : cudaSuccess;
}
template <class T>
cudaError_t host_array(am_sweep* h, T** p, size_t bytes, unsigned flags = cudaHostAllocDefault) {
  void* q = nullptr;
  cudaError_t e = cudaHostAlloc(&q, bytes, flags);
  if (e != cudaSuccess) return e;
  own(h, Owned::kPinned, q);
  *p = (T*)q;
  return cudaSuccess;
}
cudaError_t new_event(am_sweep* h, cudaEvent_t* ev, bool timed = false) {
  cudaError_t e = timed ? cudaEventCreate(ev) : cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
  if (e == cudaSuccess) own(h, Owned::kEvent, (void*)*ev);
  return e;
}
cudaError_t new_stream(am_sweep* h, cudaStream_t* s) {
  cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
  if (e == cudaSuccess) own(h, Owned::kStream, (void*)*s);
  return e;
}

// `bytes` of device memory at `src` into host memory at `dst`, after everything on the handle's stream: through pin_in,
// one synchronisation.
int read_back(am_sweep* h, void* dst, const void* src, size_t bytes) {
  AM_CUDA(h, h->pin_in.reserve(bytes));
  AM_CUDA(h, cudaMemcpyAsync(h->pin_in.p, src, bytes, cudaMemcpyDeviceToHost, h->stream));
  AM_CUDA(h, cudaStreamSynchronize(h->stream));
  memcpy(dst, h->pin_in.p, bytes);
  return AM_OK;
}

// The least key (~0 = none) that reduce(key) — min-reductions launched on the handle's stream — leaves in a word of
// dev_in that starts at ~0.
template <class Reduce>
int min_key(am_sweep* h, Reduce&& reduce, unsigned long long* out) {
  AM_CUDA(h, h->dev_in.reserve(8));
  AM_CUDA(h, cudaMemsetAsync(h->dev_in.p, 0xFF, 8, h->stream));
  AM_CUDA(h, reduce((unsigned long long*)h->dev_in.p));
  return read_back(h, out, h->dev_in.p, 8);
}

// The seconds the calendar arithmetic takes: |unix_sec| < 2^55.
bool time_ok(int64_t unix_sec) { return unix_sec < (1ll << 55) && unix_sec > -(1ll << 55); }

// Grow a pinned staging array (called under h->mu); keeps the contents.  Copies out of the
// old array may still be in flight on the copy stream: wait for them before it is freed.
cudaError_t grow_pinned(am_sweep* h, PinnedBuf& b, size_t used_bytes, size_t want_bytes, bool copies_in_flight) {
  if (want_bytes <= b.cap) return cudaSuccess;
  void* np = nullptr;
  size_t ncap = want_bytes * 2 + 65536;
  cudaError_t e = cudaHostAlloc(&np, ncap, cudaHostAllocDefault);
  if (e != cudaSuccess) return e;
  if (used_bytes) memcpy(np, b.p, used_bytes);
  if (b.p) {
    if (copies_in_flight) cudaStreamSynchronize(h->cstream);
    cudaFreeHost(b.p);
  }
  b.p = np;
  b.cap = ncap;
  return cudaSuccess;
}

// Enqueue the not-yet-copied part of a staging area on the copy stream, if the device
// twins are large enough (they are grown at drain time only).  Called under h->mu by the
// posting threads (chunk threshold) and by the drain (everything).
cudaError_t flush_staging(am_sweep* h, Staging& st, bool all, size_t upto = SIZE_MAX) {
  // ops: everything below `upto` is complete.  Without an explicit bound that is all of them, or, while
  // posting calls are still filling reserved ranges, the completed prefix.
  if (upto == SIZE_MAX) upto = st.writers ? st.done_ops : st.n_ops;
  const size_t pend = upto > st.flushed_ops ? upto - st.flushed_ops : 0;
  if (pend && (all || pend >= kFlushOps) && st.d_ops.cap >= upto * 8) {
    cudaError_t e = cudaMemcpyAsync((uint64_t*)st.d_ops.p + st.flushed_ops, (const uint64_t*)st.ops.p + st.flushed_ops,
                                    pend * 8, cudaMemcpyHostToDevice, h->cstream);
    if (e != cudaSuccess) return e;
    st.flushed_ops = upto;
    st.copy_pending = true;
  }
  const size_t pr = st.n_recs - st.flushed_recs;
  if (pr && (all || pr >= kFlushRecs) && st.d_recs.cap >= st.n_recs * sizeof(am_record_t)) {
    cudaError_t e = cudaMemcpyAsync((am_record_t*)st.d_recs.p + st.flushed_recs,
                                    (const am_record_t*)st.recs.p + st.flushed_recs, pr * sizeof(am_record_t),
                                    cudaMemcpyHostToDevice, h->cstream);
    if (e != cudaSuccess) return e;
    st.flushed_recs = st.n_recs;
    st.copy_pending = true;
  }
  return cudaSuccess;
}

// A reserved range [a, b) of the op arrays is completely staged (called under h->mu): extend the
// completed prefix, absorbing ranges that finished earlier above it.
void complete_range(Staging& st, size_t a, size_t b) {
  if (a != st.done_ops) { st.done_ranges.emplace_back(a, b); return; }
  st.done_ops = b;
  for (bool again = true; again && !st.done_ranges.empty();) {
    again = false;
    for (size_t k = 0; k < st.done_ranges.size(); ++k)
      if (st.done_ranges[k].first == st.done_ops) {
        st.done_ops = st.done_ranges[k].second;
        st.done_ranges[k] = st.done_ranges.back();
        st.done_ranges.pop_back();
        again = true;
        break;
      }
  }
}

// Make room for `n` more staged ops (and `nrec` more upsert records) in the current staging area;
// called with h->mu held through `lk`.  The pinned arrays move when they grow: calls that are
// still filling a reserved range outside the lock are waited for first.
int reserve_staging(am_sweep* h, std::unique_lock<std::mutex>& lk, size_t n, size_t nrec, Staging** out) {
  for (;;) {
    Staging& st = h->stage[h->cur];
    if (st.n_ops + n > 0x3FFFFFF0ull || st.n_recs + nrec > 0x3FFFFFF0ull) return AM_E_NOSPACE;
    const size_t want = (st.n_ops + n) * 8, want_r = (st.n_recs + nrec) * sizeof(am_record_t);
    if (st.ops.cap < want || (nrec && st.recs.cap < want_r)) {
      if (st.writers) { h->cv.wait(lk); continue; }  // (the drain may have swapped the areas meanwhile)
      AM_CUDA(h, cudaSetDevice(h->device));
      const bool inflight = st.flushed_ops || st.flushed_recs || st.copy_pending;
      AM_CUDA(h, grow_pinned(h, st.ops, st.n_ops * 8, want, inflight));
      if (nrec) AM_CUDA(h, grow_pinned(h, st.recs, st.n_recs * sizeof(am_record_t), want_r, inflight));
    }
    *out = &st;
    return AM_OK;
  }
}

// The end of a drain of n ops from `st` (with spec updates among them when `spec`): its marks cleared, and the point
// after which the device twins of `st` may be overwritten recorded.
int clear_marks(am_sweep* h, Staging& st, size_t n, bool spec, cudaStream_t s) {
  const unsigned B = 256, G = (unsigned)((n + B - 1) / B);
  auto* k = spec ? clear_marks_kernel<true> : clear_marks_kernel<false>;
  AM_CUDA(h, launch_pdl(h, k, G, B, s, h->marks, (const uint2*)st.d_ops.p, (uint32_t)n,
                        spec ? h->spec_marks : nullptr));
  AM_CUDA(h, cudaEventRecord(st.drained, s));
  st.drain_pending = true;
  return AM_OK;
}

// clear_marks of a drain that deferred it (host ticks: the sweep does not touch the marks, and the
// host waits for an event recorded BEFORE this launch — the clear is off the tick's latency)
int finish_deferred_clear(am_sweep* h, cudaStream_t s) {
  Staging* st = h->pend_clear;
  if (!st) return AM_OK;
  h->pend_clear = nullptr;
  return clear_marks(h, *st, h->pend_clear_n, h->pend_clear_spec, s);
}

// Workflow timeouts: no deadline in [first, first + n) (the segment bounds stay lower bounds: a segment reached by its
// bound finds nothing and gets its exact minimum); `all` also resets every bound.
int drop_deadlines(am_sweep* h, cudaStream_t s, uint64_t first, uint64_t n, bool all) {
  AM_CUDA(h, launch(h, fill_i64_kernel, h->sms * 8, 256, s, h->deadline + first, kNoDeadline, n));
  if (all) AM_CUDA(h, cudaMemsetAsync(h->seg_deadline, 0xFF, h->cap_padded / kRecPerWarp * 8, s));
  return AM_OK;
}

// The timeout state, allocated by the first drain that stages a non-zero wf_timeout: 24 B per slot (W 4, deadline 8,
// the list's index 4 and since 8) and 8 B per 128-slot segment.
int alloc_timeouts(am_sweep* h, cudaStream_t s) {
  const size_t cap = h->cap_padded;
  AM_CUDA(h, dev_array(h, &h->wf_timeout, cap * 4, s));
  AM_CUDA(h, dev_array(h, &h->deadline, cap * 8, s, false));
  AM_CUDA(h, dev_array(h, &h->seg_deadline, cap / kRecPerWarp * 8, s, false));
  AM_CUDA(h, dev_array(h, &h->to_idx, cap * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->to_since, cap * 8, s, false));
  AM_CUDA(h, dev_array(h, &h->to_count, 4, s));
  return drop_deadlines(h, s, 0, cap, true);
}

// Submit budget: the admission passes run while the hold is on and the admission state exists.
bool admission_on(const am_sweep* h) { return h->hold && h->adm_ctl; }

// No slot waits for admission, the FIFO is empty, the last tick's numbers are zero (the oldest second INT64_MAX).
int reset_admission(am_sweep* h, cudaStream_t s) {
  AM_CUDA(h, launch(h, fill_i64_kernel, h->sms * 8, 256, s, h->adm_wait, kNotWaiting, h->cap_padded));
  AdmCtl z{};
  z.oldest = INT64_MAX;
  AM_CUDA(h, cudaMemcpyAsync(h->adm_ctl, &z, sizeof z, cudaMemcpyHostToDevice, s));  // (pageable: copied before the return)
  return AM_OK;
}

// The admission state, allocated at the first finite budget: 21.14 B per slot of capacity (the waiting second 8, the FIFO
// and a tick's kept and new slots 12, a byte per FIFO entry, a bit of fresh submissions, 4 B per FIFO chunk).
int alloc_admission(am_sweep* h, cudaStream_t s) {
  const size_t cap = h->cap_padded, ngroups = groups_of(cap);
  AM_CUDA(h, dev_array(h, &h->adm_wait, cap * 8, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_fifo, cap * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_keep, cap * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_fresh, cap * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_cand, cap, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_sub, ngroups * kGroupWords * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_group_sub, ngroups * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_chunk, (cap / kAdmBlock + 1) * 4, s, false));
  AM_CUDA(h, dev_array(h, &h->adm_ctl, sizeof(AdmCtl), s, false));
  return reset_admission(h, s);
}

// Whether a slot waits for admission, as the waits stand after the last drain (FIFO entries whose slot stopped waiting
// do not count): one pass over the FIFO and one read-back.
int admission_waiting(am_sweep* h, bool* out) {
  *out = false;
  if (!admission_on(h)) return AM_OK;
  int rc = set_stream(h, h->stream);
  if (rc != AM_OK) return rc;
  unsigned long long key;
  rc = min_key(h, [&](unsigned long long* k) {
    return launch(h, adm_next_due_kernel, h->sms * 4, 256, h->stream, (const uint32_t*)h->adm_fifo,
                  (const int64_t*)h->adm_wait, (const AdmCtl*)h->adm_ctl, (int64_t)0, k);
  }, &key);
  if (rc == AM_OK) *out = key != ~0ull;
  return rc;
}

// The FIFO rebuilt from the waiting seconds of the swept slots, in admission order (second, then slot), on the host: a
// restore places waits anywhere in the order.  The last tick's counts become those of an empty tick with this backlog.
int rebuild_admission_fifo(am_sweep* h) {
  std::vector<int64_t> wait(h->n_records);
  if (h->n_records)
    AM_CUDA(h, cudaMemcpy(wait.data(), h->adm_wait, h->n_records * 8, cudaMemcpyDeviceToHost));
  std::vector<uint32_t> fifo;
  for (uint64_t i = 0; i < h->n_records; ++i)
    if (wait[i] != kNotWaiting) fifo.push_back((uint32_t)i);
  std::stable_sort(fifo.begin(), fifo.end(), [&](uint32_t a, uint32_t b) { return wait[a] < wait[b]; });
  if (!fifo.empty()) AM_CUDA(h, cudaMemcpy(h->adm_fifo, fifo.data(), fifo.size() * 4, cudaMemcpyHostToDevice));
  AdmCtl q{};
  q.n_fifo = q.n_deferred = fifo.size();
  q.oldest = fifo.empty() ? INT64_MAX : wait[fifo[0]];
  AM_CUDA(h, cudaMemcpy(h->adm_ctl, &q, sizeof q, cudaMemcpyHostToDevice));
  return AM_OK;
}

// A tick's admission passes, between its sweep and scan_groups_kernel, over buffer set `ts` (admission_kernels.cuh).
int launch_admission(am_sweep* h, int64_t T, const TickSet& ts, cudaStream_t s) {
  AdmParams a{};
  a.out = ts.out;
  a.n_groups = groups_of(h->n_records);
  a.n_tiles = tiles_of(h->n_records);
  a.c = h->cols;
  a.since = h->since;
  if (h->wf_timeout) {
    a.deadline = h->deadline;
    a.wf_timeout = h->wf_timeout;
    a.seg_deadline = h->seg_deadline;
  }
  a.wait = h->adm_wait;
  a.fifo = h->adm_fifo;
  a.keep = h->adm_keep;
  a.fresh = h->adm_fresh;
  a.cand = h->adm_cand;
  a.sub = h->adm_sub;
  a.group_sub = h->adm_group_sub;
  a.chunk = h->adm_chunk;
  a.ctl = h->adm_ctl;
  a.budget = h->budget;
  a.T = T;
  const unsigned grid = (unsigned)h->sms * 4;  // (the per-entry passes loop over the backlog's chunks)
  AM_CUDA(h, launch(h, adm_masks_kernel, a.n_groups, kGroupWords, s, a));
  AM_CUDA(h, launch(h, adm_check_kernel, grid, kAdmBlock, s, a));
  AM_CUDA(h, launch(h, adm_plan_kernel, 1, 1024, s, a));
  AM_CUDA(h, launch(h, adm_fifo_kernel, grid, kAdmBlock, s, a));
  AM_CUDA(h, launch(h, adm_fresh_kernel, a.n_groups, kGroupWords, s, a));
  AM_CUDA(h, launch(h, adm_merge_kernel, grid, 256, s, a));
  return AM_OK;
}

// A tick's expiry pass (expire_runs_kernel), while the hold is on and the timeout state exists.  Every tick that gets
// as far as its drain resets the timed-out list.
int expire_runs(am_sweep* h, cudaStream_t s, int64_t T) {
  h->to_ran = h->hold && h->wf_timeout;
  h->to_fetched = false;
  if (!h->to_ran) return AM_OK;
  AM_CUDA(h, cudaMemsetAsync(h->to_count, 0, 4, s));
  const uint64_t n_seg = (h->n_records + kRecPerWarp - 1) / kRecPerWarp;
  if (n_seg) {  // one lane per segment bound, one warp per 32 of them
    AM_CUDA(h, launch_pdl(h, expire_runs_kernel, (unsigned)((n_seg + 255) / 256), 256, s, h->cols, h->since,
                          h->deadline, h->seg_deadline, (uint32_t)n_seg, T, h->to_idx, h->to_since, h->to_count));
    if (h->details)  // (before note_slots_kernel: a clear bit means the slot's pair is stale)
      AM_CUDA(h, launch_pdl(h, capture_timeouts_kernel, h->sms, 256, s, h->det_applied, h->det_start,
                            (const uint32_t*)h->chg_bits, (const uint32_t*)h->to_idx, (const int64_t*)h->to_since,
                            (const uint32_t*)h->to_count));
    if (h->track)  // status changes: every timed-out run gets its Failed applied by this tick
      AM_CUDA(h, launch_pdl(h, note_slots_kernel, h->sms, 256, s, h->chg_bits, (const uint32_t*)h->to_idx,
                            (const uint32_t*)h->to_count));
  }
  return AM_OK;
}

// Status changes: the bits of slots [first, first + n) from the flags as they stand (a live record with a pending result
// is changed by the next tick), for turning tracking on and for am_sweep_load_range.
int seed_changes(am_sweep* h, cudaStream_t s, uint64_t first, uint64_t n) {
  AM_CUDA(h, launch(h, seed_changes_kernel, h->sms * 8, 256, s, h->chg_bits, (const uint32_t*)h->cols.flags, first, n));
  if (h->details)
    AM_CUDA(h, launch(h, seed_details_kernel, h->sms * 8, 256, s, h->det_applied, h->det_start,
                      (const uint32_t*)h->cols.flags, first, n));
  return AM_OK;
}

// The plane words of every segment that overlaps slots [first, first + n), the partial ones at either end included (a
// load or a restore of the range), on the handle's stream.
int rebuild_planes(am_sweep* h, uint64_t first, uint64_t n) {
  const uint64_t seg0 = first / kRecPerWarp, n_seg = (first + n + kRecPerWarp - 1) / kRecPerWarp - seg0;
  AM_CUDA(h, launch(h, build_planes_range_kernel, (unsigned)((n_seg + kWarps - 1) / kWarps), kBlock, h->stream, h->cols,
                    h->planes, (uint32_t)seg0, (uint32_t)n_seg));
  h->due_valid = false;  // (the range's ras and finishedAt were replaced: the next plain tick rebuilds the due words)
  return AM_OK;
}

// Status changes after a tick's sweep (buffer set `parity`): STOPPED in, ANOMALY out (and in closed loop every completed
// submission in), then the bits compacted into the ascending list, which clears them.  A host tick launches this behind
// the event it waits for: am_sweep_last_changes waits for it.
int list_changes(am_sweep* h, cudaStream_t s, int parity, bool closed, int64_t T) {
  h->chg_parity = parity;
  h->chg_T = T;
  h->chg_closed = closed;
  h->det_listed = h->details;
  if (h->n_records == 0) return AM_OK;  // (nothing swept: the list stays empty)
  const TickSet& ts = h->set[parity];
  const uint32_t n_tiles = tiles_of(h->n_records), n_groups = groups_of(h->n_records);
  if (h->details)
    AM_CUDA(h, launch_pdl(h, capture_sweep_kernel, (n_tiles + kWarps - 1) / kWarps, kBlock, s, h->det_applied,
                          h->det_start, (const uint32_t*)h->chg_bits, ts.out, n_tiles, closed));
  AM_CUDA(h, launch_pdl(h, note_exceptions_kernel, (n_tiles + kWarps - 1) / kWarps, kBlock, s, h->chg_bits, ts.out,
                        n_tiles, closed));
  AM_CUDA(h, launch_pdl(h, count_changes_kernel, n_groups, kGroupWords, s, h->chg_bits, (const uint32_t*)h->cols.flags,
                        h->chg_group));
  ScanParams sc{};
  sc.group_count = h->chg_group;
  sc.group_prefix = h->chg_prefix;
  sc.acc = h->chg_acc;
  sc.n_groups = n_groups;
  sc.cap = 0xFFFFFFFFu;
  AM_CUDA(h, launch_pdl(h, scan_groups_kernel, 1, 1024, s, sc));
  AM_CUDA(h, launch_pdl(h, list_changes_kernel, n_groups, kGroupWords, s, h->chg_bits, (const uint32_t*)h->chg_prefix,
                        h->chg_list));
  if (h->details)
    AM_CUDA(h, launch_pdl(h, snapshot_details_kernel, h->sms * 4, 256, s, (const uint32_t*)h->chg_list,
                          (const unsigned long long*)(h->chg_acc + 1), (const uint8_t*)h->det_applied,
                          (const int64_t*)h->det_start, h->det_e_applied, h->det_e_start));
  h->chg_listed = true;
  return AM_OK;
}

// Take buffer set `ts` for a tick on `s`: an exchange on another stream may still be reading it, and a tick_shard
// whose statistics no exchange published left them in its accumulators (they are not this tick's).
int claim_set(am_sweep* h, TickSet& ts, cudaStream_t s) {
  if (ts.consumed_pending) {
    AM_CUDA(h, cudaStreamWaitEvent(s, ts.consumed, 0));
    ts.consumed_pending = false;
  }
  if (ts.unpublished) {
    AM_CUDA(h, cudaMemsetAsync(ts.acc, 0, kNumAcc * 8, s));
    ts.unpublished = false;
  }
  return AM_OK;
}

// The due words for a kernel that writes ras or finishedAt to keep, NULL when there is nothing exact to keep.
uint32_t* due_kept(const am_sweep* h) { return h->due_valid ? h->due : nullptr; }

// Apply staged upserts / removes / results on stream `s` (called with the tick guard held).
// The staging lock is held only for the buffer swap.
int drain_staged(am_sweep* h, cudaStream_t s, const int64_t* tick_T = nullptr, bool defer_clear = false) {
  Staging* st;
  {
    std::unique_lock<std::mutex> lk(h->mu);
    st = &h->stage[h->cur];
    h->cv.wait(lk, [&] { return st->writers == 0; });  // posting calls still filling their ranges
    if (st->n_ops == 0) {
      lk.unlock();
      return tick_T ? expire_runs(h, s, *tick_T) : AM_OK;
    }
    // callers are about to append to the other area: its previous copies must have left it
    Staging& nx = h->stage[h->cur ^ 1];
    if (nx.copy_pending) {
      AM_CUDA(h, cudaEventSynchronize(nx.copied));
      nx.copy_pending = false;
    }
    // ... and the kernels of its previous drain must be done with its device twins before
    // the chunked copies of the coming events overwrite them (asynchronous ticks only)
    if (nx.drain_pending) {
      AM_CUDA(h, cudaStreamWaitEvent(h->cstream, nx.drained, 0));
      nx.drain_pending = false;
    }
    h->cur ^= 1;
  }
  // from here on `st` is private to this (single) ticking thread
  const size_t n = st->n_ops, nrec = st->n_recs;
  if (st->hwm > h->n_records) set_hwm(h, st->hwm);  // every upserted slot extends the swept range
  if (st->d_ops.cap < n * 8 || st->d_recs.cap < nrec * sizeof(am_record_t)) {
    // grow the device twins (frees synchronise) and copy everything again
    AM_CUDA(h, cudaStreamSynchronize(h->cstream));
    AM_CUDA(h, st->d_ops.reserve(n * 8));
    AM_CUDA(h, st->d_recs.reserve(nrec * sizeof(am_record_t)));
    st->flushed_ops = st->flushed_recs = 0;
  }
  AM_CUDA(h, flush_staging(h, *st, true));
  // Change details of a drain longer than a call tag's span: two post calls may carry one tag, and
  // capture_superseded_kernel tells them apart by their first op indices (pageable: copied before the return)
  const uint32_t* d_calls = nullptr;
  const uint32_t n_calls = (uint32_t)st->calls.size();
  if (h->details && n > kCallTagSpan && n_calls > 1) {
    if (st->d_calls.cap < n_calls * 4ull) {
      AM_CUDA(h, cudaStreamSynchronize(h->cstream));  // (frees synchronise)
      AM_CUDA(h, st->d_calls.reserve(n_calls * 4ull));
    }
    AM_CUDA(h, cudaMemcpyAsync(st->d_calls.p, st->calls.data(), n_calls * 4ull, cudaMemcpyHostToDevice, h->cstream));
    d_calls = (const uint32_t*)st->d_calls.p;
  }
  AM_CUDA(h, cudaEventRecord(st->copied, h->cstream));
  st->copy_pending = true;
  AM_CUDA(h, cudaStreamWaitEvent(s, st->copied, 0));
  const uint2* d_ops = (const uint2*)st->d_ops.p;
  const am_record_t* d_recs = (const am_record_t*)st->d_recs.p;
  const unsigned B = 256, G = (unsigned)((n + B - 1) / B);
  const bool spec = st->n_spec != 0;
  if (spec && !h->spec_marks) AM_CUDA(h, dev_array(h, &h->spec_marks, h->cap_padded * 4, s));
  auto* mark_ops = spec ? mark_ops_kernel<true> : mark_ops_kernel<false>;
  AM_CUDA(h, launch(h, mark_ops, G, B, s, h->marks, d_ops, (uint32_t)n, spec ? h->spec_marks : nullptr));
  if (st->n_state)
    AM_CUDA(h, launch_pdl(h, apply_state_ops_kernel, G, B, s, h->cols, h->marks, d_ops, d_recs, (uint32_t)n,
                          h->seg_dirty, due_kept(h), h->due_epoch));
  if (spec) {  // spec updates on top of the upserts: their W after the upserts' W, so a later spec update's wins
    if (st->any_wf && !h->wf_timeout) {
      const int rc = alloc_timeouts(h, s);
      if (rc != AM_OK) return rc;
    }
    if (h->wf_timeout && st->n_state)
      AM_CUDA(h, launch_pdl(h, store_wf_timeout_kernel, G, B, s, h->wf_timeout, h->marks, d_ops, d_recs, (uint32_t)n));
    AM_CUDA(h, launch_pdl(h, apply_spec_ops_kernel, G, B, s, h->cols, h->marks, (const uint32_t*)h->spec_marks, d_ops,
                          d_recs, (uint32_t)n, h->seg_dirty, h->wf_timeout, h->track ? h->chg_bits : nullptr,
                          h->details ? h->det_applied : nullptr, h->details ? h->det_start : nullptr, due_kept(h),
                          h->due_epoch));
  }
  if (st->n_state || spec) {
    // upserts, removes and spec updates may change kinds, zones and masks: rebuild the plane words of the segments
    // they touched (every drain, so a later tick sees them whichever call drained)
    auto* build_planes = spec ? build_planes_dirty_kernel<true> : build_planes_dirty_kernel<false>;
    AM_CUDA(h, launch_pdl(h, build_planes, (unsigned)((n + kWarps - 1) / kWarps), kBlock, s, h->cols, h->planes,
                          h->seg_dirty, d_ops, (uint32_t)n));
  }
  if (h->track)  // status changes: the phases of this drain that survive, and what its upserts and removes overwrote
    AM_CUDA(h, launch_pdl(h, note_ops_kernel, G, B, s, h->chg_bits, (const uint32_t*)h->cols.flags, h->marks, d_ops,
                          (uint32_t)n));
  if (h->details) {  // change details: what the surviving phases apply and the runs they end (since not yet cleared)
    AM_CUDA(h, launch_pdl(h, capture_ops_kernel, G, B, s, h->det_applied, h->det_start, h->cols,
                          (const int64_t*)(h->hold ? h->since : nullptr), (const uint32_t*)h->marks, d_ops,
                          (uint32_t)n));
    auto* superseded = spec ? capture_superseded_kernel<true> : capture_superseded_kernel<false>;
    AM_CUDA(h, launch_pdl(h, superseded, G, B, s, h->det_start, (const uint32_t*)h->marks, d_ops, (uint32_t)n, d_calls,
                          n_calls));
  }
  if (st->any_wf && !h->wf_timeout) {
    const int rc = alloc_timeouts(h, s);
    if (rc != AM_OK) return rc;
  }
  if (h->wf_timeout && st->n_state && !spec)  // (upserts with W = 0 overwrite an older W as well)
    AM_CUDA(h, launch_pdl(h, store_wf_timeout_kernel, G, B, s, h->wf_timeout, h->marks, d_ops, d_recs, (uint32_t)n));
  if (h->hold)  // a posted workflow phase or a remove ends the slot's run (an upsert keeps the hold)
    AM_CUDA(h, launch_pdl(h, clear_since_kernel, G, B, s, h->since, d_ops, (uint32_t)n));
  if (admission_on(h))  // ... and ends the slot's wait for admission (its FIFO entry is dropped at the next tick)
    AM_CUDA(h, launch_pdl(h, clear_since_kernel, G, B, s, h->adm_wait, d_ops, (uint32_t)n));
  // Workflow timeouts expire here, ahead of the result kernels: a remedy phase posted alone in this drain is then
  // applied together with the synthetic Failed, as it is behind a Failed posted after it (the remedy gate sees both).
  if (tick_T) {
    const int rc = expire_runs(h, s, *tick_T);
    if (rc != AM_OK) return rc;
  }
  // A tick's drain applies sparse results right away (apply_results_now_kernel: no second memory round trip
  // in the sweep, and the posted bits never pass through the flags as a separate step); a read's drain, or a
  // batch touching more than an eighth of the records, leaves them pending in the flags for the sweep's own
  // streaming path (apply_result_ops_kernel).
  if (tick_T && st->n_result && h->early_results && (uint64_t)st->n_result * 8 <= h->n_records) {
    TickSet& ts = h->set[h->parity];  // the buffer set of the tick being prepared
    if (int rc = claim_set(h, ts, s)) return rc;
    const bool r = h->remedy;  // (remedy runs start here; the deadline words exist with the timeout state)
    auto* apply_now = r ? apply_results_now_kernel<true> : apply_results_now_kernel<false>;
    AM_CUDA(h, launch_pdl(h, apply_now, G, B, s, h->cols, h->marks, d_ops, (uint32_t)n, *tick_T, ts.acc,
                          r ? h->since : nullptr, r ? h->deadline : nullptr,
                          r ? (const int32_t*)h->wf_timeout : nullptr, r ? h->seg_deadline : nullptr, due_kept(h),
                          h->due_epoch));
  } else if (st->n_result) {
    AM_CUDA(h, launch_pdl(h, apply_result_ops_kernel, G, B, s, h->cols.flags, h->marks, d_ops, (uint32_t)n));
  }
  if (defer_clear) {  // (the caller runs finish_deferred_clear on the same stream before anything else touches the handle)
    h->pend_clear = st;
    h->pend_clear_n = n;
    h->pend_clear_spec = spec;
  } else {
    const int rc = clear_marks(h, *st, n, spec, s);
    if (rc != AM_OK) return rc;
  }
  st->n_ops = st->n_recs = st->flushed_ops = st->flushed_recs = 0;
  st->done_ops = 0;
  st->done_ranges.clear();
  st->calls.clear();
  st->n_state = st->n_result = st->n_spec = 0;
  st->any_wf = false;
  st->hwm = 0;
  return AM_OK;
}

// The prologue of a call that is not a tick (tick guard held): on the handle's stream, after every upsert, remove
// and result staged before it.
int begin_call(am_sweep* h) {
  const int rc = set_stream(h, h->stream);
  return rc != AM_OK ? rc : drain_staged(h, h->stream);
}

// dev_in / pin_in for an on-demand kernel: `out_bytes` of results at the start, then (when `idx` is given) the n
// slots as u32, copied to the device on the handle's stream.  *d_idx = that device copy, or NULL without `idx`.
int stage_indices(am_sweep* h, size_t out_bytes, uint64_t n, const uint64_t* idx, const uint32_t** d_idx) {
  AM_CUDA(h, h->pin_in.reserve(out_bytes + (idx ? n * 4 : 0)));
  AM_CUDA(h, h->dev_in.reserve(out_bytes + (idx ? n * 4 : 0)));
  *d_idx = nullptr;
  if (!idx) return AM_OK;
  uint32_t* hidx = (uint32_t*)((char*)h->pin_in.p + out_bytes);
  for (uint64_t k = 0; k < n; ++k) hidx[k] = (uint32_t)idx[k];
  uint32_t* didx = (uint32_t*)((char*)h->dev_in.p + out_bytes);
  AM_CUDA(h, cudaMemcpyAsync(didx, hidx, n * 4, cudaMemcpyHostToDevice, h->stream));
  *d_idx = didx;
  return AM_OK;
}

// Where the rebuilt list goes: HBM (device-resident pipelines), mapped host memory (host
// ticks) or nowhere (am_sweep_tick_shard: the exchange rebuilds the global list).
struct ListOut {
  void* idx = nullptr;      // u32 local indices
  uint8_t* act = nullptr;
  uint64_t cap = 0;
  uint32_t* count = nullptr;          // min(n_emitted, cap), device memory, may be NULL
  am_tick_stats_t* stats = nullptr;   // device or mapped host memory, may be NULL
  bool expand = true;
};

// Copy `bytes` of `src` into `u` on `s`.  Stream-ordered: a kernel still reading the previous contents runs before
// the copy (every device operation of a handle is ordered).
int upload(am_sweep* h, Upload& u, size_t full, const void* src, size_t bytes, cudaStream_t s) {
  if (!u.dev) AM_CUDA(h, dev_array(h, &u.dev, full, s));
  if (!u.pin) AM_CUDA(h, host_array(h, &u.pin, full));  // full size at once: the pinned array never moves under a copy
  if (!u.copied) AM_CUDA(h, new_event(h, &u.copied));
  if (u.pending) AM_CUDA(h, cudaEventSynchronize(u.copied));  // the previous copy has left the pinned array
  memcpy(u.pin, src, bytes);
  AM_CUDA(h, cudaMemcpyAsync(u.dev, u.pin, bytes, cudaMemcpyHostToDevice, s));
  AM_CUDA(h, cudaEventRecord(u.copied, s));
  u.pending = true;
  return AM_OK;
}

// The zones' UTC offsets at T on the device.  Per tick: one uncontended lock for the registry version
// and two compares; the offsets themselves are recomputed (tz_eval.h, host) and copied — a few hundred
// bytes — only when a zone was registered or T left the window in which no zone changes its offset.
int refresh_zones(am_sweep* h, int64_t T, cudaStream_t s) {
  if (amsweep_tz::snapshot(nullptr, nullptr, nullptr) == h->tz_version && T >= h->tz_lo && T < h->tz_hi) return AM_OK;
  std::vector<int32_t> offs;
  int64_t until = 0;
  bool aligned = true;
  const uint64_t v = amsweep_tz::offsets_at(T, &offs, &until, &aligned);
  h->tz_version = v;
  h->tz_n = (uint32_t)offs.size();
  h->tz_lo = T;
  h->tz_hi = until;
  h->tz_aligned = aligned;
  if (h->tz_n <= 1) {  // nothing registered: every T is fine until the registry grows
    h->tz_lo = INT64_MIN;
    h->tz_hi = INT64_MAX;
    return AM_OK;
  }
  // allocated once, for every id a record can carry; entries of zones not registered stay zero
  if (!h->tz_table) AM_CUDA(h, dev_array(h, &h->tz_table, (amsweep_tz::kMaxZones + 1) * sizeof(TickWords), s));
  return upload(h, h->tz_off, (amsweep_tz::kMaxZones + 1) * sizeof(int32_t), offs.data(), offs.size() * sizeof(int32_t), s);
}

// A catch-up tick's window (P, T] as calendar boxes per zone.  Computed before anything of the tick happens,
// so that AM_E_RANGE leaves the handle as it was.  `any` false: the tick is a plain one (no previous tick,
// T <= P, no bit, or no minute start in the window in any zone).
struct WindowPlan {
  std::vector<TickWords> boxes;  // [n_zones][kWindowBoxes]
  uint32_t n_zones = 0;
  bool any = false;
};

int plan_window(am_sweep* h, int64_t T, uint32_t mode, WindowPlan* w) {
  w->any = false;
  if (!(mode & AM_SWEEP_CATCH_UP) || !h->has_prev || T <= h->prev_T) return AM_OK;
  if (T - h->prev_T > 86400) {
    h->last_error = "AM_SWEEP_CATCH_UP: more than a day since the previous tick";
    return AM_E_RANGE;
  }
  bool steady = false;
  if (!amsweep_tz::window_boxes(h->prev_T, T, &w->boxes, &w->n_zones, &steady)) {
    h->last_error = "AM_SWEEP_CATCH_UP: a time zone splits the window into too many calendar boxes";
    return AM_E_RANGE;
  }
  // The ticker's normal cadence: T is the window's only minute start in every zone (T on the UTC minute, P at most a
  // minute back, every offset whole minutes and unchanged in the window).  The plain on-minute tick at T is then the
  // same tick, and reads the planes instead of the 40 B of canonical masks per record.
  int64_t sec_of_min = T % 60;
  if (sec_of_min < 0) sec_of_min += 60;
  if (steady && sec_of_min == 0 && T - h->prev_T <= 60) return AM_OK;
  for (const TickWords& b : w->boxes) w->any |= b.sec0 != 0;
  return AM_OK;
}

// The sweep variant of a tick: a row per loop mode, a column per way the masks are read (not at all, the planes of
// T's minute, the canonical masks against a catch-up window's boxes).  These are the 22 instantiations of
// sweep_tick_kernel there are.  Three combinations have none and never get here: closed loop with the hold on (refused
// before the drain, and run_ticks refuses the hold), a window with the planes (launch_tick sets `masks` only
// without a window) and the due words with a window (due_tick takes them only without one).
using SweepFn = void (*)(const SweepParams);
SweepFn sweep_variant(bool closed, bool masks, bool window, bool hold, bool timeout, bool remedy, int due) {
  static constexpr SweepFn kVariants[8][3] = {
      // open loop
      {sweep_tick_kernel<false, false>, sweep_tick_kernel<false, true>, sweep_tick_kernel<false, false, true>},
      // closed loop
      {sweep_tick_kernel<true, false>, sweep_tick_kernel<true, true>, sweep_tick_kernel<true, false, true>},
      // hold in flight (open loop)
      {sweep_tick_kernel<false, false, false, true>, sweep_tick_kernel<false, true, false, true>,
       sweep_tick_kernel<false, false, true, true>},
      // ... and workflow timeouts
      {sweep_tick_kernel<false, false, false, true, true>, sweep_tick_kernel<false, true, false, true, true>,
       sweep_tick_kernel<false, false, true, true, true>},
      // hold in flight with the remedy hold
      {sweep_tick_kernel<false, false, false, true, false, true>, sweep_tick_kernel<false, true, false, true, false, true>,
       sweep_tick_kernel<false, false, true, true, false, true>},
      // ... and workflow timeouts
      {sweep_tick_kernel<false, false, false, true, true, true>, sweep_tick_kernel<false, true, false, true, true, true>,
       sweep_tick_kernel<false, false, true, true, true, true>},
      // open loop from the due words, and open loop building them (no window, no hold: due_tick)
      {sweep_tick_kernel<false, false, false, false, false, false, kDueRead>,
       sweep_tick_kernel<false, true, false, false, false, false, kDueRead>, nullptr},
      {sweep_tick_kernel<false, false, false, false, false, false, kDueBuild>,
       sweep_tick_kernel<false, true, false, false, false, false, kDueBuild>, nullptr}};
  return kVariants[due ? 5 + due : hold ? 2 + timeout + 2 * remedy : closed][window ? 2 : masks];
}

// The DUE of a tick's sweep variant.  An open-loop tick without a window or the hold, on a handle that has not handed
// out ras or finishedAt, reads the due words when they are exact for every slot it sweeps and T lies in their epoch's
// window; otherwise it builds them (kDueBuild, epoch T - 2^31: the tick reads ras and finishedAt as without the words and
// writes every swept slot's word, so a rebuild costs no launch).  Any other tick runs a variant that may write
// finishedAt without its word: the words are dropped.
int due_tick(am_sweep* h, int64_t T, bool plain, uint32_t n_tiles, cudaStream_t s, int* due) {
  *due = kDueOff;
  if (!plain || h->due_exposed.load(std::memory_order_relaxed)) {
    h->due_valid = false;
    return AM_OK;
  }
  const uint64_t end = (uint64_t)n_tiles * kTile;
  if (h->due_valid && T >= h->due_epoch && T - h->due_epoch < kDueSpan && end <= h->due_end) {
    *due = kDueRead;
    return AM_OK;
  }
  if (!h->due) AM_CUDA(h, dev_array(h, &h->due, h->cap_padded * 4, s, false));
  h->due_epoch = T - kDueEpochLead;
  h->due_end = end;
  h->due_valid = true;  // (from this tick's sweep on)
  *due = kDueBuild;
  return AM_OK;
}

int launch_tick(am_sweep* h, int64_t T, uint32_t mode, const ListOut& o, cudaStream_t s, const WindowPlan* win = nullptr) {
  if (h->n_records == 0) {
    // nothing to sweep: publish zeros without a launch
    if (o.stats) AM_CUDA(h, cudaMemsetAsync(o.stats, 0, sizeof(am_tick_stats_t), s));
    if (o.count) AM_CUDA(h, cudaMemsetAsync(o.count, 0, 4, s));
    return AM_OK;
  }
  TickSet& ts = h->set[h->parity];
  if (int rc = claim_set(h, ts, s)) return rc;
  SweepParams p{};
  p.c = h->cols;
  p.n_records = h->n_records;
  p.shard_base = h->shard_base;
  p.seed = h->seed;
  p.T = T;
  p.words = tick_words_from_unix(T);
  p.n_tiles = tiles_of(h->n_records);
  p.mode = mode;
  p.out = ts.out;
  p.acc = ts.acc;
  {  // named time zones: one UTC offset per zone, valid at T
    const int rc = refresh_zones(h, T, s);
    if (rc != AM_OK) return rc;
  }
  // off the minute no 5-field schedule can fire: the mask columns are not read.  (A zone whose UTC
  // offset is not a whole number of minutes — historical local mean times — moves the local minute
  // boundary: every tick then reads the masks.)
  int64_t sec_of_min = T % 60;
  if (sec_of_min < 0) sec_of_min += 60;
  // A catch-up tick reads the canonical masks against the window's boxes instead of planes and zone words.
  const bool window = win && win->any;
  const bool masks = !window && (sec_of_min == 0 || (mode & AM_SWEEP_FULL_SCAN) || (h->tz_n > 1 && !h->tz_aligned));
  if (window) {  // zones registered after the plan keep zero entries (sec0 = 0): no box, not due
    const int rc = upload(h, h->win_boxes, (size_t)(amsweep_tz::kMaxZones + 1) * kWindowBoxes * sizeof(TickWords),
                          win->boxes.data(), win->boxes.size() * sizeof(TickWords), s);
    if (rc != AM_OK) return rc;
    p.tz_table = (const TickWords*)h->win_boxes.dev;
  }
  if (masks && h->tz_n > 1) {  // the tick's wall clock per zone, from the cached offsets
    AM_CUDA(h, launch_pdl(h, tz_words_kernel, (h->tz_n + 63) / 64, 64, s, (const int32_t*)h->tz_off.dev, h->tz_table, T,
                          h->tz_n));
    p.tz_table = h->tz_table;
  }
  if (masks) {  // the six planes of T's UTC fields
    const CivilTime ct = civil_from_unix(T);
    auto plane = [&](int k) { return (const uint32_t*)(h->planes.w + (size_t)k * h->planes.words); };
    p.pl.minute = plane(kPlaneMinute + ct.min);
    p.pl.hour = plane(kPlaneHour + ct.hour);
    p.pl.dom = plane(kPlaneDom + ct.dom);
    p.pl.month = plane(kPlaneMonth + ct.month);
    p.pl.dow = plane(kPlaneDow + ct.dow);
    p.pl.star = plane(kPlaneStar);
  }
  const bool closed = (mode & AM_SWEEP_CLOSED_LOOP) != 0;
  int due = kDueOff;
  if (int rc = due_tick(h, T, !closed && !window && !h->hold, p.n_tiles, s, &due)) return rc;
  if (h->profiling) AM_CUDA(h, cudaEventRecord(h->evp[0], s));
  const bool timeout = h->hold && h->wf_timeout;
  if (h->hold) p.since = h->since;  // hold in flight: the variants that read and write since
  if (timeout) {                    // ... and workflow timeouts: the variants that also set deadlines
    p.wf_timeout = h->wf_timeout;
    p.deadline = h->deadline;
    p.seg_deadline = h->seg_deadline;
  }
  if (due) {
    p.due = h->due;
    p.due_t = (uint32_t)(T - h->due_epoch);
    p.due_epoch = h->due_epoch;
  }
  const SweepFn sweep = sweep_variant(closed, masks, window, h->hold, timeout, h->remedy, due);
  // A single-stream tick's sweep launches early and hides behind its predecessor (the previous tick's publish, the
  // drain).  am_sweep_tick_shard's is a plain launch: an early-launched sweep could park its CTAs on every SM ahead
  // of the previous tick's exchange on the other stream; measured at two GPUs it made no difference to the step, so
  // the simpler form stays.
  AM_CUDA(h, o.expand ? launch_pdl(h, sweep, p.n_tiles, kBlock, s, p) : launch(h, sweep, p.n_tiles, kBlock, s, p));
  if (h->profiling) AM_CUDA(h, cudaEventRecord(h->evp[1], s));
  if (admission_on(h)) {  // the submit budget cuts the sweep's output in place (profiling: counted in the rest)
    const int rc = launch_admission(h, T, ts, s);
    if (rc != AM_OK) return rc;
  }
  ScanParams sc{};
  sc.group_count = ts.out.group_count;
  sc.group_prefix = ts.out.group_prefix;
  sc.acc = ts.acc;
  sc.out_count = o.count;
  sc.n_groups = groups_of(h->n_records);
  sc.cap = (uint32_t)(o.cap > 0xFFFFFFFFull ? 0xFFFFFFFFull : o.cap);
  AM_CUDA(h, launch_pdl(h, scan_groups_kernel, 1, 1024, s, sc));
  if (o.expand) {
    ExpandParams e{};
    e.src[0].bitmap = ts.out.bitmap;
    e.src[0].group_prefix = ts.out.group_prefix;
    e.src[0].tile_exc = ts.out.tile_exc;
    e.src[0].exc_seg = ts.out.exc_seg;
    e.src[0].base = 0;  // local indices
    e.src[0].n_groups = sc.n_groups;
    e.src[0].n_tiles = p.n_tiles;
    e.out_idx = o.idx;
    e.out_act = o.act;
    e.acc = ts.acc;
    e.stats_base = h->shard_base;
    e.cap = o.idx ? o.cap : 0;
    e.world = 1;
    e.stats_rank = 0;
    e.idx_bytes = 4;
    AM_CUDA(h, launch_pdl(h, expand_kernel, dim3(sc.n_groups, 1), kExpandThreads, s, e));
    AM_CUDA(h, launch_pdl(h, publish_kernel, 1, 32, s, ts.acc, o.stats, h->n_records));
  }
  if (h->profiling) { AM_CUDA(h, cudaEventRecord(h->evp[2], s)); h->profiled = true; }
  h->parity ^= 1;
  return AM_OK;
}

// A host tick's list goes to mapped pinned memory (u32 indices, then u8 actions), its statistics to the mapped struct.
int host_list_out(am_sweep* h, ListOut* o) {
  const uint64_t entries = h->n_records;
  if (entries > h->host_out_entries) {
    const uint64_t want = (entries + entries / 4 + 4095) / 4096 * 4096;
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    AM_CUDA(h, h->host_out.reserve(want * 5, cudaHostAllocMapped));
    h->host_out_entries = want;
  }
  if (h->host_out_entries) {
    void* d = nullptr;
    AM_CUDA(h, cudaHostGetDevicePointer(&d, h->host_out.p, 0));
    o->idx = d;
    o->act = (uint8_t*)d + h->host_out_entries * 4;
    o->cap = h->host_out_entries;
  }
  o->stats = h->d_stats_mapped;
  return AM_OK;
}

// Which entry point a tick came through: a host tick (am_sweep_tick, am_sweep_tick_view) writes the list into
// h->host_out and waits for it, a device tick writes it where the caller said, a shard tick leaves it to the exchange.
enum class TickKind { kHost, kDevice, kShard };

// One tick of the handle, with the tick guard held and T in range.  Refusals come before anything happens (nothing
// drained, P unchanged): closed loop with the hold on (a closed-loop record completes in the tick that submits it, so
// nothing is ever in flight to hold), then the catch-up plan.  P, the second of the previous tick, moves only when
// the tick succeeds.
int run_tick(am_sweep* h, int64_t T, uint32_t mode, cudaStream_t s, TickKind kind, ListOut o = {},
             am_tick_stats_t* stats = nullptr) {
  if (h->hold && (mode & AM_SWEEP_CLOSED_LOOP)) {
    h->last_error = "AM_SWEEP_CLOSED_LOOP while the hold in flight is on";
    return AM_E_INVAL;
  }
  WindowPlan win;
  int rc = plan_window(h, T, mode, &win);
  if (rc != AM_OK) return rc;
  rc = set_stream(h, s);
  if (rc != AM_OK) return rc;
  const bool host = kind == TickKind::kHost;
  h->chg_listed = h->chg_fetched = false;  // (every tick that drains resets the list of status changes)
  rc = drain_staged(h, s, &T, /*defer_clear=*/host);
  struct ClearOnExit {  // whatever happens below, the marks are cleared before the handle is used again
    am_sweep* h;
    cudaStream_t s;
    ~ClearOnExit() { (void)finish_deferred_clear(h, s); }
  } clear_on_exit{h, s};
  if (rc != AM_OK) return rc;
  if (kind == TickKind::kShard) {
    if (h->n_records == 0) return AM_E_INVAL;  // an empty shard has nothing to exchange
    o.expand = false;
  }
  if (host) {
    rc = host_list_out(h, &o);
    if (rc != AM_OK) return rc;
    AM_CUDA(h, cudaEventRecord(h->ev0, s));
  }
  const int parity = (int)h->parity;
  rc = launch_tick(h, T, mode, o, s, &win);
  if (rc != AM_OK) return rc;
  if (host) {
    AM_CUDA(h, cudaEventRecord(h->ev1, s));
    rc = finish_deferred_clear(h, s);  // behind the event the host waits for
    if (rc != AM_OK) return rc;
  }
  if (h->track) {  // (a host tick: behind that event as well)
    rc = list_changes(h, s, parity, (mode & AM_SWEEP_CLOSED_LOOP) != 0, T);
    if (rc != AM_OK) return rc;
  }
  if (host) {  // one synchronisation
    AM_CUDA(h, cudaEventSynchronize(h->ev1));
    float ms = 0;
    AM_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    h->last_ms = ms;
    am_tick_stats_t st = *h->h_stats;
    st.n_records = h->n_records;
    h->host_n = st.n_emitted;
    if (stats) *stats = st;
  } else if (kind == TickKind::kShard) {
    h->last_shard_parity = parity;
    h->set[parity].unpublished = true;
  }
  h->has_prev = true;
  h->prev_T = T;
  ++h->ticks;
  return AM_OK;
}

// The prologue of a run of ticks (am_sweep_run_ticks, am_sweep_simulate; tick guard held, refusals made): on the
// handle's stream, the staged calls drained (as tick *tick_T's drain when given), the run's seed.  A run's ticks list
// no timed-out runs and no status changes.
int begin_run(am_sweep* h, const int64_t* tick_T, uint64_t seed) {
  int rc = set_stream(h, h->stream);
  if (rc != AM_OK) return rc;
  h->to_ran = false;
  h->chg_listed = h->chg_fetched = false;
  rc = drain_staged(h, h->stream, tick_T);
  if (rc != AM_OK) return rc;
  h->seed = seed;
  return AM_OK;
}

// The device rows of a run of n ticks: n am_tick_stats_t and, for a simulation, n am_sim_tick_t (4 accumulators each)
// after them.  One allocation, freed on every return.
struct RunRows {
  am_tick_stats_t* stats = nullptr;
  unsigned long long* sim = nullptr;
  size_t bytes = 0;
  ~RunRows() { cudaFree(stats); }
  cudaError_t alloc(uint64_t n, bool with_sim) {
    bytes = n * (sizeof(am_tick_stats_t) + (with_sim ? sizeof(am_sim_tick_t) : 0));
    const cudaError_t e = cudaMalloc((void**)&stats, bytes);
    if (e == cudaSuccess && with_sim) sim = reinterpret_cast<unsigned long long*>(stats + n);
    return e;
  }
};

// Ticks per pass of a blocked run: AMSWEEP_BLOCK_TICKS in [1, kMaxBlockTicks], else kDefaultBlockTicks.
uint64_t block_ticks() {
  if (const char* e = getenv("AMSWEEP_BLOCK_TICKS")) {
    const long v = atol(e);
    if (v >= 1 && v <= kMaxBlockTicks) return (uint64_t)v;
  }
  return kDefaultBlockTicks;
}

// Temporal blocking (sweep_block.cuh): the n ticks from T0 in blocks of up to block_ticks() ticks, one pass over the
// columns each.  A block never spans an instant at which a registered zone changes its UTC offset (the kernel holds one
// offset per zone for the whole block).  Per block, `b`'s BlockParams part is filled in and launch_block(b, k, grid)
// launches the caller's instantiation for the block that starts at tick k, returning the launch error.
template <class P, class Launch>
int run_blocks(am_sweep* h, int64_t T0, uint64_t n, am_tick_stats_t* stats, P b, Launch&& launch_block) {
  const uint64_t per_block = block_ticks();
  h->due_valid = false;  // (the blocked kernels write finishedAt without the due words)
  const unsigned grid = (unsigned)((h->n_records + kBlockRecords - 1) / kBlockRecords);
  for (uint64_t k = 0; k < n;) {
    const int64_t T = T0 + (int64_t)k;
    const int rc = refresh_zones(h, T, h->stream);
    if (rc != AM_OK) return rc;
    uint64_t K = n - k < per_block ? n - k : per_block;
    if (h->tz_n > 1 && h->tz_hi < T + (int64_t)K) K = (uint64_t)(h->tz_hi - T);  // (tz_hi > T after the refresh)
    b.c = h->cols;
    b.n_records = h->n_records;
    b.shard_base = h->shard_base;
    b.seed = h->seed;
    b.T0 = T;
    b.K = (uint32_t)K;
    b.tz_off = h->tz_n > 1 ? (const int32_t*)h->tz_off.dev : nullptr;
    b.stats = reinterpret_cast<unsigned long long*>(stats + k);
    AM_CUDA(h, launch_block(b, k, grid));
    k += K;
  }
  return AM_OK;
}

// A run of n ticks from T0 once begin_run is done: its rows (zeroed when blocked or simulated: the kernels accumulate
// into them), ev0, ticks(rows) (the entry's own ticks), ev1, one synchronisation, the rows copied out (the sim rows
// when sim_out is given), last_ms, n_records in every row of a blocked run, and P committed on success.  With
// tracking on, a run that got as far as its rows seeds the change bits again from the flags whatever happened: its
// ticks applied what its drain noted.
template <class Ticks>
int run_rows(am_sweep* h, int64_t T0, uint64_t n, bool blocked, bool with_sim, am_tick_stats_t* stats_out,
             am_sim_tick_t* sim_out, Ticks&& ticks) {
  RunRows rows;
  AM_CUDA(h, rows.alloc(n, with_sim));
  int rc = [&]() -> int {
    if (blocked || with_sim) AM_CUDA(h, cudaMemsetAsync(rows.stats, 0, rows.bytes, h->stream));
    AM_CUDA(h, cudaEventRecord(h->ev0, h->stream));
    const int trc = ticks(rows);
    if (trc != AM_OK) return trc;
    AM_CUDA(h, cudaEventRecord(h->ev1, h->stream));
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    AM_CUDA(h, cudaMemcpy(stats_out, rows.stats, n * sizeof(am_tick_stats_t), cudaMemcpyDeviceToHost));
    if (sim_out) AM_CUDA(h, cudaMemcpy(sim_out, rows.sim, n * sizeof(am_sim_tick_t), cudaMemcpyDeviceToHost));
    float ms = 0;
    AM_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    h->last_ms = ms;
    if (blocked)  // (a tick's publish_kernel writes its row's n_records)
      for (uint64_t k = 0; k < n; ++k) stats_out[k].n_records = h->n_records;
    h->has_prev = true;
    h->prev_T = T0 + (int64_t)n - 1;
    h->ticks += n;
    return AM_OK;
  }();
  if (h->track) {
    const int rs = seed_changes(h, h->stream, 0, h->cap_padded);
    if (rc == AM_OK) rc = rs;
  }
  return rc;
}

}  // namespace

namespace amsweep {
bool shard_last_tick(am_sweep* h, ShardTick* out) {
  if (!h || h->last_shard_parity < 0) return false;
  const TickSet& ts = h->set[h->last_shard_parity];
  out->out = ts.out;
  out->acc = ts.acc;
  out->shard_base = h->shard_base;
  out->n_records = h->n_records;
  out->n_groups = groups_of(h->n_records);
  out->n_tiles = tiles_of(h->n_records);
  out->parity = h->last_shard_parity;
  out->device = h->device;
  return true;
}
int shard_order_consumer(am_sweep* h, cudaStream_t s) { return wait_last(h, s); }
int shard_launch_expand(am_sweep* h, const ExpandParams& e, uint32_t groups_x, uint32_t world_y, cudaStream_t s) {
  AM_CUDA(h, launch(h, expand_kernel, dim3(groups_x, world_y), kExpandThreads, s, e));
  return AM_OK;
}
int shard_launch_publish(am_sweep* h, unsigned long long* acc, am_tick_stats_t* out_stats, uint64_t n_records,
                         cudaStream_t s) {
  AM_CUDA(h, launch(h, publish_kernel, 1, 32, s, acc, out_stats, n_records));
  return AM_OK;
}
int shard_mark_consumed(am_sweep* h, int parity, cudaStream_t s) {
  TickSet& ts = h->set[parity & 1];
  AM_CUDA(h, cudaEventRecord(ts.consumed, s));
  ts.consumed_pending = true;
  ts.unpublished = false;  // (the exchange's publish_kernel re-armed the accumulators)
  return AM_OK;
}
}  // namespace amsweep

extern "C" {

const char* am_last_error_detail(const am_sweep_t* h) {
  if (h) return h->last_error.c_str();
  static thread_local std::string copy;  // stable storage for the returned pointer
  std::lock_guard<std::mutex> lk(g_create_mu);
  copy = g_create_error;
  return copy.c_str();
}

int am_sweep_create(am_sweep_t** out, int device_id, uint64_t capacity, uint64_t shard_base) {
  if (!out || capacity == 0 || capacity > 0xFFFFF000ull) return AM_E_INVAL;
  *out = nullptr;
  am_sweep* none = nullptr;
  int ndev = 0;
  AM_CUDA(none, cudaGetDeviceCount(&ndev));
  if (device_id < 0 || device_id >= ndev) {
    set_create_error("no such CUDA device");
    return AM_E_DEVICE;
  }
  AM_CUDA(none, cudaSetDevice(device_id));
  am_sweep* h = new (std::nothrow) am_sweep();
  if (!h) return AM_E_NOMEM;
  h->device = device_id;
  h->capacity = capacity;
  h->cap_padded = (capacity + kTile - 1) / kTile * kTile;
  h->shard_base = shard_base;
  if (const char* e = getenv("AMSWEEP_EARLY_RESULTS")) h->early_results = atoi(e) != 0;  // (A/B of the two result paths)
  int rc = [&]() -> int {
    AM_CUDA(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, device_id));
    AM_CUDA(h, new_stream(h, &h->stream));
    AM_CUDA(h, new_stream(h, &h->cstream));
    for (cudaEvent_t* e : {&h->ev_last, &h->stage[0].copied, &h->stage[0].drained, &h->stage[1].copied,
                           &h->stage[1].drained, &h->set[0].consumed, &h->set[1].consumed})
      AM_CUDA(h, new_event(h, e));
    for (cudaEvent_t* e : {&h->ev0, &h->ev1, &h->evp[0], &h->evp[1], &h->evp[2]}) AM_CUDA(h, new_event(h, e, true));
    for (int k = 0; k < 16; ++k) AM_CUDA(h, dev_array(h, col_slot(h->cols, k), h->cap_padded * kColElem[k], h->stream));
    AM_CUDA(h, launch(h, fill_u32_kernel, h->sms * 8, 256, h->stream, h->cols.flags, AM_F_TOMBSTONE, h->cap_padded));
    // the mask planes: every slot is a tombstone, no record has a plane bit
    h->planes.words = h->cap_padded / 32;
    AM_CUDA(h, dev_array(h, &h->planes.w, kPlanes * h->planes.words * 4, h->stream));
    AM_CUDA(h, dev_array(h, &h->seg_dirty, h->cap_padded / kRecPerWarp * 4, h->stream));
    const size_t ntiles = h->cap_padded / kTile;
    const size_t ngroups = (ntiles + kGroupTiles - 1) / kGroupTiles;
    for (TickSet& ts : h->set) {
      TickOut& t = ts.out;
      // bitmap words past the last tile of the last group are never written: they stay zero
      AM_CUDA(h, dev_array(h, &t.bitmap, ngroups * kGroupWords * 4, h->stream));
      AM_CUDA(h, dev_array(h, &t.group_count, ngroups * 4, h->stream));
      AM_CUDA(h, dev_array(h, &t.group_prefix, (ngroups + 1) * 4, h->stream));
      AM_CUDA(h, dev_array(h, &t.tile_exc, ntiles * 4, h->stream));
      AM_CUDA(h, dev_array(h, &t.exc_seg, h->cap_padded * 4, h->stream));  // expand_kernel prefetches past the counts
      AM_CUDA(h, dev_array(h, &ts.acc, kNumAcc * 8, h->stream));
    }
    AM_CUDA(h, dev_array(h, &h->marks, h->cap_padded * 12, h->stream));
    for (int b = 0; b < 2; ++b) {
      AM_CUDA(h, dev_array(h, &h->due_idx[b], h->cap_padded * 4, h->stream, false));
      AM_CUDA(h, dev_array(h, &h->due_action[b], h->cap_padded, h->stream, false));
    }
    AM_CUDA(h, host_array(h, &h->h_stats, sizeof(am_tick_stats_t), cudaHostAllocMapped));
    memset(h->h_stats, 0, sizeof(am_tick_stats_t));
    AM_CUDA(h, cudaHostGetDevicePointer((void**)&h->d_stats_mapped, h->h_stats, 0));
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    return AM_OK;
  }();
  if (rc != AM_OK) {
    set_create_error(h->last_error);
    am_sweep_destroy(h);
    return rc;
  }
  *out = h;
  return AM_OK;
}

void am_sweep_destroy(am_sweep_t* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();  // ticks may have been issued on caller streams
  for (const Owned& o : h->owned) {
    if (o.kind == Owned::kDevice) cudaFree(o.p);
    else if (o.kind == Owned::kPinned) cudaFreeHost(o.p);
    else if (o.kind == Owned::kEvent) cudaEventDestroy((cudaEvent_t)o.p);
    else cudaStreamDestroy((cudaStream_t)o.p);
  }
  for (Staging& st : h->stage) {
    st.ops.release(); st.recs.release();
    st.d_ops.release(); st.d_recs.release(); st.d_calls.release();
  }
  h->host_out.release();
  h->pin_in.release(); h->dev_in.release();
  delete h;
}

uint64_t am_sweep_size(const am_sweep_t* h) { return h ? __atomic_load_n(&h->n_records, __ATOMIC_RELAXED) : 0; }
uint64_t am_sweep_capacity(const am_sweep_t* h) { return h ? h->capacity : 0; }
int am_sweep_device(const am_sweep_t* h) { return h ? h->device : -1; }
double am_sweep_last_kernel_ms(const am_sweep_t* h) { return h ? h->last_ms : -1.0; }
uint64_t am_sweep_launch_count(const am_sweep_t* h) { return h ? h->launches.load(std::memory_order_relaxed) : 0; }
void* am_sweep_column_ptr(am_sweep_t* h, int column) {
  if (!h || column < 0 || column >= 16) return nullptr;
  if (column == 5 || column == 7) h->due_exposed.store(true, std::memory_order_relaxed);  // ras, finished_at
  return *col_slot(h->cols, column);
}
int am_sweep_set_profiling(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  h->profiling = on != 0;
  h->profiled = false;
  return AM_OK;
}
int am_sweep_last_profile(am_sweep_t* h, double* sweep_ms, double* rest_ms) {
  if (!h || !h->profiled) return AM_E_INVAL;
  AM_CUDA(h, cudaSetDevice(h->device));
  AM_CUDA(h, cudaEventSynchronize(h->evp[2]));
  float a = 0, b = 0;
  AM_CUDA(h, cudaEventElapsedTime(&a, h->evp[0], h->evp[1]));
  AM_CUDA(h, cudaEventElapsedTime(&b, h->evp[1], h->evp[2]));
  if (sweep_ms) *sweep_ms = a;
  if (rest_ms) *rest_ms = b;
  return AM_OK;
}
void* am_sweep_stream(am_sweep_t* h) { return h ? (void*)h->stream : nullptr; }
int am_sweep_set_seed(am_sweep_t* h, uint64_t seed) {
  if (!h) return AM_E_INVAL;
  h->seed = seed;
  return AM_OK;
}

int am_sweep_load_range(am_sweep_t* h, uint64_t first, uint64_t n, const am_record_cols_t* cols) {
  if (!h || !cols || first + n > h->capacity || first + n < first) return AM_E_INVAL;
  if (n == 0) return AM_OK;
  if (cols->flags && amsweep_host::unknown_zones(n, cols->flags, 1, (uint32_t)amsweep_tz::count())) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  // a load is a call in the per-slot order: upserts, removes and results staged before it are applied first, so
  // the load overwrites them (a result is left pending in the flags, which the load replaces; a posted workflow
  // phase has released its slot's hold in this drain all the same)
  int rc = begin_call(h);
  if (rc != AM_OK) return rc;
  for (int k = 0; k < 16; ++k) {
    char* dst = (char*)*col_slot(h->cols, k) + first * kColElem[k];
    const void* src = *cols_member(cols, k);
    if (src) AM_CUDA(h, cudaMemcpyAsync(dst, src, n * kColElem[k], cudaMemcpyHostToDevice, h->stream));
    else AM_CUDA(h, cudaMemsetAsync(dst, 0, n * kColElem[k], h->stream));
  }
  rc = rebuild_planes(h, first, n);
  if (rc != AM_OK) return rc;
  if (h->hold)  // loaded records have nothing in flight
    AM_CUDA(h, launch(h, fill_i64_kernel, h->sms * 8, 256, h->stream, h->since + first, kNotInFlight, n));
  if (admission_on(h))  // ... and wait for nothing
    AM_CUDA(h, launch(h, fill_i64_kernel, h->sms * 8, 256, h->stream, h->adm_wait + first, kNotWaiting, n));
  if (h->wf_timeout) {  // am_record_cols_t has no timeout column: loaded slots have none, and no deadline
    AM_CUDA(h, cudaMemsetAsync(h->wf_timeout + first, 0, n * 4, h->stream));
    rc = drop_deadlines(h, h->stream, first, n, false);
    if (rc != AM_OK) return rc;
  }
  if (h->track) {  // the load replaced whatever the drains had noted for the range
    rc = seed_changes(h, h->stream, first, n);
    if (rc != AM_OK) return rc;
  }
  AM_CUDA(h, cudaStreamSynchronize(h->stream));
  if (first + n > h->n_records) set_hwm(h, first + n);
  return AM_OK;
}

int am_sweep_set_hold_in_flight(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if ((on != 0) == h->hold) return AM_OK;
  if (on) {  // starts with nothing in flight
    int rc = set_stream(h, h->stream);
    if (rc != AM_OK) return rc;
    if (!h->since) AM_CUDA(h, dev_array(h, &h->since, h->cap_padded * sizeof(int64_t), h->stream, false));
    AM_CUDA(h, launch(h, fill_i64_kernel, h->sms * 8, 256, h->stream, h->since, kNotInFlight, h->cap_padded));
    if (h->wf_timeout) {  // (the deadlines of runs from before the hold was turned off)
      rc = drop_deadlines(h, h->stream, 0, h->cap_padded, true);
      if (rc != AM_OK) return rc;
    }
  }
  if (h->adm_ctl) {  // every wait for admission ends
    int rc = set_stream(h, h->stream);
    if (rc == AM_OK) rc = reset_admission(h, h->stream);
    if (rc != AM_OK) return rc;
  }
  h->budget = UINT64_MAX;
  h->hold = on != 0;
  if (!on) h->remedy = false;  // (the since words are refilled when the hold is turned on again)
  return AM_OK;
}

int am_sweep_set_submit_budget(am_sweep_t* h, uint64_t per_tick) {
  if (!h) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->hold) {
    h->last_error = "am_sweep_set_submit_budget while the hold in flight is off";
    return AM_E_INVAL;
  }
  if (per_tick != UINT64_MAX && !h->adm_ctl) {
    int rc = set_stream(h, h->stream);
    if (rc == AM_OK) rc = alloc_admission(h, h->stream);
    if (rc != AM_OK) return rc;
  }
  h->budget = per_tick;
  return AM_OK;
}

int am_sweep_last_admission(am_sweep_t* h, am_admission_t* out) {
  if (!h || !out) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->adm_ctl) {
    h->last_error = "am_sweep_last_admission: the handle never had a finite submit budget";
    return AM_E_INVAL;
  }
  int rc = set_stream(h, h->stream);  // (after a device tick: waits for it)
  if (rc != AM_OK) return rc;
  AdmCtl q{};
  AM_CUDA(h, cudaMemcpyAsync(&q, h->adm_ctl, sizeof q, cudaMemcpyDeviceToHost, h->stream));
  AM_CUDA(h, cudaStreamSynchronize(h->stream));
  out->n_candidates = q.n_candidates;
  out->n_admitted = q.n_admitted;
  out->n_deferred = q.n_deferred;
  out->oldest_deferred = q.oldest;
  return AM_OK;
}

int am_sweep_set_hold_remedy(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->hold) {
    h->last_error = "am_sweep_set_hold_remedy while the hold in flight is off";
    return AM_E_INVAL;
  }
  if ((on != 0) == h->remedy) return AM_OK;
  if (!on) {  // every remedy run ends (the segment bounds stay lower bounds)
    int rc = set_stream(h, h->stream);
    if (rc != AM_OK) return rc;
    AM_CUDA(h, launch(h, release_remedy_runs_kernel, h->sms * 8, 256, h->stream, h->since, h->deadline, h->cap_padded));
  }
  h->remedy = on != 0;
  return AM_OK;
}

int am_sweep_set_track_changes(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if ((on != 0) == h->track) return AM_OK;
  h->chg_listed = h->chg_fetched = false;
  if (on) {  // 4.125 B per slot of capacity at the first enable; every enable starts from the flags as they stand
    int rc = set_stream(h, h->stream);
    if (rc != AM_OK) return rc;
    if (!h->chg_acc) {  // (the last of them: an enable that failed half-way allocates again)
      const size_t ngroups = groups_of(h->cap_padded);
      AM_CUDA(h, dev_array(h, &h->chg_bits, ngroups * kGroupWords * 4, h->stream));
      AM_CUDA(h, dev_array(h, &h->chg_list, h->cap_padded * 4, h->stream, false));
      AM_CUDA(h, dev_array(h, &h->chg_group, ngroups * 4, h->stream));
      AM_CUDA(h, dev_array(h, &h->chg_prefix, (ngroups + 1) * 4, h->stream));
      AM_CUDA(h, dev_array(h, &h->chg_acc, kNumAcc * 8, h->stream));
    }
    rc = seed_changes(h, h->stream, 0, h->cap_padded);
    if (rc != AM_OK) return rc;
  }
  h->track = on != 0;
  if (!on) h->details = false;
  return AM_OK;
}

int am_sweep_set_change_details(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->track) {
    h->last_error = "am_sweep_set_change_details while tracking is off";
    return AM_E_INVAL;
  }
  if ((on != 0) == h->details) return AM_OK;
  if (on) {  // 18 B per slot of capacity at the first enable; the staged calls first, so that what they post is pending
    int rc = begin_call(h);
    if (rc != AM_OK) return rc;
    if (!h->det_e_start) {  // (the last of them: an enable that failed half-way allocates again)
      AM_CUDA(h, dev_array(h, &h->det_applied, h->cap_padded, h->stream, false));
      AM_CUDA(h, dev_array(h, &h->det_start, h->cap_padded * 8, h->stream, false));
      AM_CUDA(h, dev_array(h, &h->det_e_applied, h->cap_padded, h->stream, false));
      AM_CUDA(h, dev_array(h, &h->det_e_start, h->cap_padded * 8, h->stream, false));
    }
    AM_CUDA(h, launch(h, seed_details_kernel, h->sms * 8, 256, h->stream, h->det_applied, h->det_start,
                      (const uint32_t*)h->cols.flags, (uint64_t)0, h->cap_padded));
  }
  h->details = on != 0;
  return AM_OK;
}

namespace {
// am_sweep_upsert (kind kOpUpsert: the swept range grows to the highest slot) and am_sweep_update_spec (kOpSpec): n
// records for slots idx, staged as one op each and a copy of the record.  A refusal stages nothing.
int stage_records(am_sweep_t* h, uint64_t n, const uint64_t* idx, const am_record_t* recs, uint32_t kind) {
  if (!h || (n && (!idx || !recs))) return AM_E_INVAL;
  if (n == 0) return AM_OK;
  if (amsweep_host::unknown_zones(n, &recs[0].flags, sizeof(am_record_t) / sizeof(uint32_t), (uint32_t)amsweep_tz::count()))
    return AM_E_INVAL;
  bool any_wf = false;
  for (uint64_t k = 0; k < n; ++k) {
    if (recs[k].wf_timeout < 0) return AM_E_RANGE;  // (nothing staged)
    any_wf |= recs[k].wf_timeout != 0;
  }
  std::unique_lock<std::mutex> lk(h->mu);
  Staging* stp = nullptr;
  if (int rc = reserve_staging(h, lk, n, n, &stp)) return rc;
  Staging& st = *stp;
  AM_CUDA(h, cudaSetDevice(h->device));
  // nothing is committed (counters unchanged) when a slot is out of range
  if (amsweep_host::stage_slots(n, idx, h->capacity, kind | (uint32_t)st.n_recs, 1u, (uint64_t*)st.ops.p + st.n_ops))
    return AM_E_RANGE;
  am_record_t* dst = (am_record_t*)st.recs.p + st.n_recs;
  uint64_t hwm = st.hwm;
  for (uint64_t k = 0; k < n; ++k) {
    dst[k] = recs[k];
    dst[k].flags &= ~AM_F_TOMBSTONE;
    if (idx[k] + 1 > hwm) hwm = idx[k] + 1;
  }
  if (kind == kOpUpsert) st.hwm = hwm;  // (a spec update of a slot that was never upserted does nothing)
  st.any_wf |= any_wf;
  complete_range(st, st.n_ops, st.n_ops + n);
  st.n_ops += n; st.n_recs += n;
  (kind == kOpUpsert ? st.n_state : st.n_spec) += (uint32_t)n;
  AM_CUDA(h, flush_staging(h, st, false));
  return AM_OK;
}
}  // namespace

int am_sweep_upsert(am_sweep_t* h, uint64_t n, const uint64_t* idx, const am_record_t* recs) {
  return stage_records(h, n, idx, recs, kOpUpsert);
}

int am_sweep_update_spec(am_sweep_t* h, uint64_t n, const uint64_t* idx, const am_record_t* recs) {
  return stage_records(h, n, idx, recs, kOpSpec);
}

int am_sweep_remove(am_sweep_t* h, uint64_t n, const uint64_t* idx) {
  if (!h || (n && !idx)) return AM_E_INVAL;
  if (n == 0) return AM_OK;
  std::unique_lock<std::mutex> lk(h->mu);
  Staging* stp = nullptr;
  if (int rc = reserve_staging(h, lk, n, 0, &stp)) return rc;
  Staging& st = *stp;
  AM_CUDA(h, cudaSetDevice(h->device));
  if (amsweep_host::stage_slots(n, idx, h->capacity, kOpRemove, 0u, (uint64_t*)st.ops.p + st.n_ops)) return AM_E_RANGE;
  complete_range(st, st.n_ops, st.n_ops + n);
  st.n_ops += n;
  st.n_state += (uint32_t)n;
  AM_CUDA(h, flush_staging(h, st, false));
  return AM_OK;
}

int am_sweep_post_result(am_sweep_t* h, uint64_t n, const uint64_t* idx, const uint8_t* phase,
                         const uint8_t* remedy_phase) {
  if (!h || (n && (!idx || !phase))) return AM_E_INVAL;
  if (n == 0) return AM_OK;
  // Reserve a range of the op arrays under the lock, fill it outside: the controller's workers
  // (hcc.go:170-188) post concurrently and the per-entry pass is the cost of a post.  Per slot the
  // call order is the reservation order.
  std::unique_lock<std::mutex> lk(h->mu);
  Staging* stp = nullptr;
  if (int rc = reserve_staging(h, lk, n, 0, &stp)) return rc;
  Staging& st = *stp;
  const size_t a = st.n_ops;
  st.calls.push_back((uint32_t)a);
  st.n_ops += n;
  st.n_result += (uint32_t)n;
  ++st.writers;  // the drain and any growth of the arrays now wait for this call
  uint64_t* const oo = (uint64_t*)st.ops.p + a;
  lk.unlock();
  // validate and stage in vectorised passes of one copy chunk each; a single large post hands every
  // finished chunk to the copy stream before staging the next (when no other call is staging).
  // phase -> flag bits: {none, Succeeded, Failed} -> {0, PENDING_OK, PENDING_FAIL}
  // Every entry carries the call's tag (its first op index, mod 2^22; capture_superseded_kernel): the entries of one
  // call see the in-flight state from before the call.  (A drain of more than 2^22 ops also uploads st.calls.)
  const uint32_t kind = kOpResult | (((uint32_t)a << kCallTagShift) & kCallTagMask);
  unsigned bad = 0;
  cudaError_t ce = cudaSuccess;
  for (uint64_t off = 0; off < n && !bad; off += kFlushOps) {
    const uint64_t m = n - off < kFlushOps ? n - off : kFlushOps;
    bad = amsweep_host::stage_results(m, idx + off, phase + off, remedy_phase ? remedy_phase + off : nullptr, h->capacity,
                                      kind, oo + off);
    if (!bad && off + m < n) {
      lk.lock();
      if (st.writers == 1 && ce == cudaSuccess && cudaSetDevice(h->device) == cudaSuccess)
        ce = flush_staging(h, st, false, a + off + m);  // everything below is complete: this call is the only one staging
      lk.unlock();
    }
  }
  // nothing of a call with a bad entry takes effect: its range is already part of the sequence (later
  // calls may have reserved behind it), so it becomes ops that mark and set nothing
  if (bad)
    for (uint64_t k = 0; k < n; ++k) oo[k] = (uint64_t)kOpResult << 32;
  lk.lock();
  complete_range(st, a, a + n);
  // Hand the completed prefix to the copy stream, a chunk at a time, even while other calls are staging.
  // The range is claimed under the lock; the copy is issued outside it (a copy call under the lock
  // serialised every worker behind the CUDA API), while this call still
  // counts as a writer — the drain, which records the "copied" event, waits for it.
  size_t c_lo = 0, c_hi = 0;
  if (ce == cudaSuccess && st.done_ops > st.flushed_ops && st.done_ops - st.flushed_ops >= kFlushOps && st.d_ops.cap >= st.done_ops * 8) {
    c_lo = st.flushed_ops;
    c_hi = st.done_ops;
    st.flushed_ops = c_hi;
    st.copy_pending = true;
  }
  const uint64_t* src = (const uint64_t*)st.ops.p;  // (the array cannot move while this call is a writer)
  lk.unlock();
  if (c_hi > c_lo && (ce = cudaSetDevice(h->device)) == cudaSuccess)
    ce = cudaMemcpyAsync((uint64_t*)st.d_ops.p + c_lo, src + c_lo, (c_hi - c_lo) * 8, cudaMemcpyHostToDevice, h->cstream);
  lk.lock();
  if (--st.writers == 0) h->cv.notify_all();
  if (bad) return (bad & 1u) ? AM_E_RANGE : AM_E_INVAL;
  AM_CUDA(h, ce);
  return AM_OK;
}

// The last tick's lists are read in pages: of n entries, those from `offset` on are left (*n_out), min(left, cap) are
// copied (*ncopy); AM_E_RANGE past the end (nothing copied), AM_E_NOSPACE when more are left than fit.
static int list_page(uint64_t n, uint64_t offset, uint64_t cap, uint64_t* n_out, uint64_t* ncopy) {
  if (offset > n) return AM_E_RANGE;
  const uint64_t left = n - offset;
  *ncopy = left < cap ? left : cap;
  if (n_out) *n_out = left;
  return left > cap ? AM_E_NOSPACE : AM_OK;
}

// Entries [offset, ...) of the last tick's host list, widened into the caller's (Go) memory.
static int copy_host_list(am_sweep_t* h, uint64_t offset, uint64_t* due_idx, uint32_t* due_action, uint64_t cap,
                          uint64_t* n_out) {
  uint64_t ncopy;
  const int page = list_page(h->host_n, offset, cap, n_out, &ncopy);
  if (page == AM_E_RANGE) return page;
  if (ncopy)
    amsweep_host::widen_list(ncopy, h->shard_base, (const uint32_t*)h->host_out.p + offset,
                             (const uint8_t*)h->host_out.p + h->host_out_entries * 4 + offset, due_idx, due_action);
  return page;
}

int am_sweep_tick(am_sweep_t* h, int64_t unix_sec, uint32_t mode, uint64_t* due_idx,
                  uint32_t* due_action, uint64_t cap, uint64_t* n_out, am_tick_stats_t* stats) {
  if (!h || (cap && (!due_idx || !due_action))) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  int rc = run_tick(h, unix_sec, mode, h->stream, TickKind::kHost, {}, stats);
  if (rc != AM_OK) return rc;
  return copy_host_list(h, 0, due_idx, due_action, cap, n_out);
}

int am_sweep_tick_view(am_sweep_t* h, int64_t unix_sec, uint32_t mode, am_tick_view_t* view,
                       am_tick_stats_t* stats) {
  if (!h || !view) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  int rc = run_tick(h, unix_sec, mode, h->stream, TickKind::kHost, {}, stats);
  if (rc != AM_OK) return rc;
  view->idx_local = (const uint32_t*)h->host_out.p;
  view->action = h->host_out.p ? (const uint8_t*)h->host_out.p + h->host_out_entries * 4 : nullptr;
  view->n = h->host_n;
  view->shard_base = h->shard_base;
  return AM_OK;
}

int am_sweep_last_list(am_sweep_t* h, uint64_t offset, uint64_t* due_idx, uint32_t* due_action,
                       uint64_t cap, uint64_t* n_out) {
  if (!h || (cap && (!due_idx || !due_action))) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  return copy_host_list(h, offset, due_idx, due_action, cap, n_out);
}

int am_sweep_tick_device(am_sweep_t* h, int64_t unix_sec, uint32_t mode, void* d_due_idx,
                         void* d_due_action, uint64_t cap, void* d_count, void* d_stats,
                         void* cuda_stream) {
  if (!h || (cap && (!d_due_idx || !d_due_action))) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  // expand_kernel stores 16-B quads of indices and 4-B words of actions, scan_groups_kernel a u32 count and
  // publish_kernel u64 statistics: a misaligned store would end the kernel with an error that takes the whole
  // CUDA context down.  Refused before anything happens (nothing drained, P unchanged).
  if (((uintptr_t)d_due_idx & 15u) || ((uintptr_t)d_due_action & 3u) || ((uintptr_t)d_count & 3u) ||
      ((uintptr_t)d_stats & 7u)) {
    h->last_error = "am_sweep_tick_device: d_due_idx must be 16-B aligned, d_due_action and d_count 4-B, d_stats 8-B";
    return AM_E_INVAL;
  }
  const ListOut o{d_due_idx, (uint8_t*)d_due_action, cap, (uint32_t*)d_count, (am_tick_stats_t*)d_stats};
  return run_tick(h, unix_sec, mode, (cudaStream_t)cuda_stream, TickKind::kDevice, o);  // NULL == CUDA default stream
}

int am_sweep_tick_shard(am_sweep_t* h, int64_t unix_sec, uint32_t mode, void* cuda_stream) {
  if (!h) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  return run_tick(h, unix_sec, mode, (cudaStream_t)cuda_stream, TickKind::kShard);
}

int am_sweep_run_ticks(am_sweep_t* h, int64_t unix_sec0, uint64_t n_ticks, uint32_t mode,
                       uint64_t seed, am_tick_stats_t* stats_out) {
  if (!h || !stats_out || (mode & AM_SWEEP_CATCH_UP)) return AM_E_INVAL;
  if (n_ticks == 0) return AM_OK;
  if (n_ticks > (1ull << 24)) return AM_E_INVAL;
  if (!time_ok(unix_sec0) || !time_ok(unix_sec0 + (int64_t)n_ticks)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (h->hold) {  // (neither the blocked kernel nor the run's plain ticks keep the hold: refused, nothing happens)
    h->last_error = "am_sweep_run_ticks while the hold in flight is on";
    return AM_E_INVAL;
  }
  // A blocked run publishes no tick's accumulators: its drain leaves posted results pending in the flags,
  // and the block kernel applies them at its first tick (and counts them in that tick's row).
  const int rc = begin_run(h, (mode & AM_SWEEP_BLOCKED) ? nullptr : &unix_sec0, seed);
  if (rc != AM_OK) return rc;
  const bool blocked = (mode & AM_SWEEP_BLOCKED) != 0 && h->n_records != 0;  // (an empty shard runs tick by tick)
  return run_rows(h, unix_sec0, n_ticks, blocked, false, stats_out, nullptr, [&](const RunRows& rows) -> int {
    if (blocked)
      return run_blocks(h, unix_sec0, n_ticks, rows.stats, BlockParams{}, [&](const BlockParams& b, uint64_t, unsigned grid) {
        auto* k = (mode & AM_SWEEP_CLOSED_LOOP) ? sweep_block_kernel<true> : sweep_block_kernel<false>;
        return launch(h, k, grid, kBlockThreads, h->stream, b);
      });
    for (uint64_t k = 0; k < n_ticks; ++k) {
      const ListOut o{h->due_idx[k & 1], h->due_action[k & 1], h->cap_padded, nullptr, rows.stats + k};
      const int trc = launch_tick(h, unix_sec0 + (int64_t)k, mode, o, h->stream);
      if (trc != AM_OK) return trc;
    }
    return AM_OK;
  });
}

int am_sweep_simulate(am_sweep_t* h, int64_t unix_sec0, uint64_t n_ticks, uint32_t mode, uint64_t seed,
                      const am_sim_params_t* params, am_tick_stats_t* stats_out, am_sim_tick_t* sim_out) {
  if (!h || !stats_out || !params || (mode & ~(AM_SWEEP_BLOCKED | AM_SWEEP_FULL_SCAN))) return AM_E_INVAL;
  if (params->wf_min < 1 || params->wf_max < params->wf_min || params->remedy_min < 1 ||
      params->remedy_max < params->remedy_min || n_ticks > (1ull << 24))
    return AM_E_INVAL;
  if (!time_ok(unix_sec0) || !time_ok(unix_sec0 + (int64_t)n_ticks)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->hold || !h->remedy) {  // (only the configuration with both holds is simulated: refused, nothing happens)
    h->last_error = "am_sweep_simulate needs the hold in flight and the remedy hold on";
    return AM_E_INVAL;
  }
  if (mode & AM_SWEEP_BLOCKED) {  // (the blocked kernel has no admission)
    bool waiting = false;
    const int brc = admission_waiting(h, &waiting);
    if (brc != AM_OK) return brc;
    if (waiting || h->budget != UINT64_MAX) {
      h->last_error = "am_sweep_simulate: AM_SWEEP_BLOCKED with a finite submit budget or checks waiting for admission";
      return AM_E_INVAL;
    }
  }
  if (n_ticks == 0) return AM_OK;
  // The staged calls come first; their results stay pending in the flags for the first tick (after its simulated posts,
  // which only ever replace a slot's bit group, as a later post_result would).
  int rc = begin_run(h, nullptr, seed);
  if (rc != AM_OK) return rc;
  const SimDraw q{seed, params->wf_min, params->wf_max - params->wf_min + 1, params->remedy_min,
                  params->remedy_max - params->remedy_min + 1};
  const bool blocked = (mode & AM_SWEEP_BLOCKED) != 0;
  if (!blocked && !h->sim_end) AM_CUDA(h, dev_array(h, &h->sim_end, h->cap_padded / kRecPerWarp * 8, h->stream, false));
  rc = run_rows(h, unix_sec0, n_ticks, blocked, true, stats_out, sim_out, [&](const RunRows& rows) -> int {
    if (blocked) {  // sweep_block_kernel<false, true>; an empty shard launches nothing
      if (h->n_records == 0) return AM_OK;
      SimBlockParams sb{};
      sb.since = h->since;
      if (h->wf_timeout) {
        sb.deadline = h->deadline;
        sb.wf_timeout = h->wf_timeout;
        sb.seg_deadline = h->seg_deadline;
      }
      sb.q = q;
      return run_blocks(h, unix_sec0, n_ticks, rows.stats, sb, [&](SimBlockParams& b, uint64_t k, unsigned grid) {
        b.sim = rows.sim + k * 4;
        return launch(h, sweep_block_kernel<false, true>, grid, kBlockThreads, h->stream, b);
      });
    }
    // Tick by tick: the completion pass, then the tick (expiry pass and sweep), then the bounds of the runs it started
    // and the tick's counts.
    const uint64_t n_seg = (h->n_records + kRecPerWarp - 1) / kRecPerWarp;
    const int64_t earliest = params->wf_min < params->remedy_min ? params->wf_min : params->remedy_min;
    AM_CUDA(h, cudaMemsetAsync(h->sim_end, 0xFF, h->cap_padded / kRecPerWarp * 8, h->stream));
    if (h->n_records)
      AM_CUDA(h, launch(h, sim_bounds_kernel, (unsigned)((h->n_records + 255) / 256), 256, h->stream, h->cols,
                        (const int64_t*)h->since, h->sim_end, h->n_records, q, h->shard_base));
    for (uint64_t k = 0; k < n_ticks; ++k) {
      const int64_t T = unix_sec0 + (int64_t)k;
      if (n_seg)
        AM_CUDA(h, launch_pdl(h, sim_complete_kernel, (unsigned)((n_seg + 255) / 256), 256, h->stream, h->cols,
                              h->since, h->sim_end, (uint32_t)n_seg, T, q, h->shard_base));
      int trc = expire_runs(h, h->stream, T);
      if (trc != AM_OK) return trc;
      const int parity = (int)h->parity;
      const ListOut o{h->due_idx[k & 1], h->due_action[k & 1], h->cap_padded, nullptr, rows.stats + k};
      trc = launch_tick(h, T, mode & AM_SWEEP_FULL_SCAN, o, h->stream);
      if (trc != AM_OK) return trc;
      if (n_seg)
        AM_CUDA(h, launch_pdl(h, sim_note_starts_kernel, (unsigned)((n_seg + 255) / 256), 256, h->stream,
                              (const uint32_t*)h->set[parity].out.bitmap, h->sim_end, (uint32_t)n_seg, T + earliest));
      AM_CUDA(h, launch_pdl(h, sim_count_kernel, h->sms * 8, 256, h->stream, h->cols, (const int64_t*)h->since,
                            h->n_records, (const int64_t*)(h->to_ran ? h->to_since : nullptr),
                            (const uint32_t*)(h->to_ran ? h->to_count : nullptr), rows.sim + k * 4));
    }
    return AM_OK;
  });
  h->to_ran = false;  // (the timed-out lists are empty afterwards, as the list of status changes is)
  return rc;
}

static int read_impl(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx, am_record_cols_t* out);

int am_sweep_repeat_after_sec(am_sweep_t* h, int64_t unix_sec, uint64_t first, uint64_t n, int64_t* out) {
  if (!h || (n && !out)) return AM_E_INVAL;
  if (first + n > h->capacity || first + n < first || n > 0xFFFFFFFFull) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  if (n == 0) return AM_OK;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  int rc = begin_call(h);
  if (rc != AM_OK) return rc;
  AM_CUDA(h, h->dev_in.reserve(n * 8));
  AM_CUDA(h, launch(h, next_fire_kernel, (unsigned)((n + 127) / 128), 128, h->stream, h->cols, (uint32_t)first,
                    (uint32_t)n, unix_sec, (int64_t*)h->dev_in.p));
  rc = read_back(h, out, h->dev_in.p, n * 8);
  if (rc != AM_OK) return rc;
  {  // schedules bound to a named time zone (marked kZoneBoundMark): Next() on the host
    std::vector<uint64_t> zi;
    for (uint64_t k = 0; k < n; ++k) if (out[k] == kZoneBoundMark) zi.push_back(first + k);
    if (!zi.empty()) {
      std::vector<uint64_t> mi(zi.size()), hr(zi.size()), dm(zi.size()), mo(zi.size()), dw(zi.size());
      std::vector<uint32_t> fl(zi.size());
      am_record_cols_t c{};
      c.minute = mi.data(); c.hour = hr.data(); c.dom = dm.data(); c.month = mo.data(); c.dow = dw.data(); c.flags = fl.data();
      const int rrc = read_impl(h, 0, zi.size(), zi.data(), &c);
      if (rrc != AM_OK) return rrc;
      for (size_t k = 0; k < zi.size(); ++k) {
        am_cron_t cr{mi[k], hr[k], dm[k], mo[k], dw[k], 0, AM_CRON_SPEC, (int32_t)(fl[k] >> AM_F_TZ_SHIFT)};
        out[zi[k] - first] = am_cron_repeat_after_sec(&cr, unix_sec);
      }
    }
  }
  return AM_OK;
}

int am_sweep_next_due(am_sweep_t* h, int64_t unix_sec, int64_t* next_out) {
  if (!h || !next_out) return AM_E_INVAL;
  if (!time_ok(unix_sec)) return AM_E_RANGE;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  int rc = begin_call(h);
  if (rc != AM_OK) return rc;
  *next_out = INT64_MAX;  // nothing will ever be due (empty shard, only tombstones / exhausted schedules)
  if (h->n_records == 0) return AM_OK;
  // Zone-bound schedules fire on their zone's minute.  While every offset is a whole number of minutes up
  // to the next UTC minute, that is not before the next UTC minute; an offset with seconds (local mean
  // time, e.g. Africa/Monrovia -0:44:30 until 1972) moves the local minute anywhere: then T + 1.
  rc = refresh_zones(h, unix_sec + 1, h->stream);
  if (rc != AM_OK) return rc;
  const int64_t next_minute = unix_sec + 60 - ((unix_sec % 60) + 60) % 60;
  const int64_t zone_due = (h->tz_aligned && h->tz_hi >= next_minute) ? next_minute : unix_sec + 1;
  unsigned long long key;
  rc = min_key(h, [&](unsigned long long* k) {
    cudaError_t e = launch(h, next_due_kernel, h->sms * 8, 256, h->stream, h->cols,
                           (const int64_t*)(h->hold ? h->since : nullptr),
                           (const int64_t*)(h->hold ? h->deadline : nullptr), h->n_records, unix_sec, zone_due, k);
    if (e == cudaSuccess && admission_on(h))  // a check still waiting for admission is due at the next second
      e = launch(h, adm_next_due_kernel, h->sms * 4, 256, h->stream, (const uint32_t*)h->adm_fifo,
                 (const int64_t*)h->adm_wait, (const AdmCtl*)h->adm_ctl, unix_sec, k);
    return e;
  }, &key);
  if (rc != AM_OK) return rc;
  if (key != ~0ull) *next_out = (int64_t)(key ^ (1ull << 63));
  return AM_OK;
}

int am_sweep_read(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx,
                  am_record_cols_t* out) {
  if (!h || !out) return AM_E_INVAL;
  if (n == 0) return AM_OK;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  const int rc = begin_call(h);  // a read observes every upsert / remove / result staged before it
  return rc != AM_OK ? rc : read_impl(h, first, n, idx, out);
}

}  // extern "C"

namespace {
// The slots of a per-slot call: [first, first + n) inside the capacity without `idx`, else every idx[k] (AM_E_RANGE
// for one past it); at most 2^32 - 1 of them either way.
int check_slots(const am_sweep* h, uint64_t first, uint64_t n, const uint64_t* idx) {
  if (n > 0xFFFFFFFFull || (!idx && (first + n > h->capacity || first + n < first))) return AM_E_INVAL;
  if (idx)
    for (uint64_t k = 0; k < n; ++k)
      if (idx[k] >= h->capacity) return AM_E_RANGE;
  return AM_OK;
}

// The per-slot states (AM_SEL_*) behind am_sweep_in_flight, _remedy_in_flight, _deferred and am_sweep_select: whether
// the handle has the state on (every slot reads INT64_MIN while it is off) ...
bool state_on(const am_sweep* h, uint32_t state) {
  return state == AM_SEL_WAITING ? admission_on(h) : h->hold && (state == AM_SEL_IN_FLIGHT || h->remedy);
}
// ... and the values of the slots first + k (d_idx NULL) or first + d_idx[k], k < n, into d_out on the handle's stream.
cudaError_t launch_values(am_sweep* h, uint32_t state, uint64_t first, const uint32_t* d_idx, uint64_t n, int64_t* d_out) {
  const unsigned grid = (unsigned)((n + 255) / 256);
  if (state == AM_SEL_WAITING)
    return launch(h, adm_gather_kernel, grid, 256, h->stream, (const int64_t*)h->adm_wait, (uint32_t)first, d_idx,
                  (uint32_t)n, d_out);
  return launch(h, in_flight_kernel, grid, 256, h->stream, h->cols, (const int64_t*)h->since, (uint32_t)first, d_idx,
                (uint32_t)n, d_out, state == AM_SEL_REMEDY_IN_FLIGHT);
}

// The path of every per-slot query: nothing for n == 0, the slots refused before the tick guard, then the guard and
// the drain (posted results, removes and loads by now release holds and end waits), then run(state_on(h, state)).
template <class Run>
int slot_query(am_sweep* h, uint32_t state, uint64_t first, uint64_t n, const uint64_t* idx, Run&& run) {
  if (n == 0) return AM_OK;
  int rc = check_slots(h, first, n, idx);
  if (rc != AM_OK) return rc;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  rc = begin_call(h);
  return rc != AM_OK ? rc : run(state_on(h, state));
}

// am_sweep_in_flight, _remedy_in_flight and _deferred: one i64 per slot, INT64_MIN everywhere while the state is off.
int query_slots(am_sweep* h, uint32_t state, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* out) {
  if (!h || (n && !out)) return AM_E_INVAL;
  return slot_query(h, state, first, n, idx, [&](bool on) {
    if (!on) {
      for (uint64_t k = 0; k < n; ++k) out[k] = INT64_MIN;
      return AM_OK;
    }
    const uint32_t* d_idx;
    int rc = stage_indices(h, n * 8, n, idx, &d_idx);
    if (rc != AM_OK) return rc;
    AM_CUDA(h, launch_values(h, state, idx ? 0 : first, d_idx, n, (int64_t*)h->dev_in.p));
    return read_back(h, out, h->dev_in.p, n * 8);
  });
}

int sel_alloc(am_sweep* h) {
  if (h->sel_acc) return AM_OK;
  const size_t ngroups = groups_of(h->cap_padded);
  AM_CUDA(h, dev_array(h, &h->sel_bits, ngroups * kGroupWords * 4, h->stream, false));
  AM_CUDA(h, dev_array(h, &h->sel_group, ngroups * 4, h->stream, false));
  AM_CUDA(h, dev_array(h, &h->sel_prefix, (ngroups + 1) * 4, h->stream, false));
  AM_CUDA(h, dev_array(h, &h->sel_list, h->cap_padded * 4, h->stream, false));
  AM_CUDA(h, dev_array(h, &h->sel_acc, 2 * 8, h->stream, false));  // (the last: the others exist once it does)
  return AM_OK;
}
}  // namespace

extern "C" {

int am_sweep_in_flight(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* since_out) {
  return query_slots(h, AM_SEL_IN_FLIGHT, first, n, idx, since_out);
}

int am_sweep_remedy_in_flight(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* started_out) {
  return query_slots(h, AM_SEL_REMEDY_IN_FLIGHT, first, n, idx, started_out);
}

int am_sweep_deferred(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx, int64_t* since_out) {
  return query_slots(h, AM_SEL_WAITING, first, n, idx, since_out);
}

// The mark pass writes the range's bitmap, group counts and accumulators; with cap > 0 the scan and the compaction
// list every match (relative to first) and the values of the first m = min(cap, n) list entries are gathered.  The
// entries past the matches are zeroed first, so that the gather reads slot `first` for them.  One synchronisation
// brings back the accumulators and m entries of the list and the values.
int am_sweep_select(am_sweep_t* h, uint32_t state, uint64_t first, uint64_t n, int64_t before, uint64_t* idx,
                    int64_t* value, uint64_t cap, uint64_t* n_match, int64_t* oldest) {
  if (!h || state < AM_SEL_IN_FLIGHT || state > AM_SEL_WAITING || !n_match || !oldest || (cap && (!idx || !value)))
    return AM_E_INVAL;
  *n_match = 0;
  *oldest = INT64_MAX;
  return slot_query(h, state, first, n, nullptr, [&](bool on) {
    if (!on) return AM_OK;
    int rc = sel_alloc(h);
    if (rc != AM_OK) return rc;
    const uint32_t n_groups = groups_of(n);
    const uint64_t m = std::min(cap, n);
    AM_CUDA(h, cudaMemsetAsync(h->sel_acc, 0xFF, 8, h->stream));
    AM_CUDA(h, cudaMemsetAsync(h->sel_acc + 1, 0, 8, h->stream));
    const bool waiting = state == AM_SEL_WAITING;
    AM_CUDA(h, launch(h, select_mark_kernel, n_groups, kGroupWords, h->stream, h->cols,
                      (const int64_t*)(waiting ? nullptr : h->since), (const int64_t*)(waiting ? h->adm_wait : nullptr),
                      state == AM_SEL_REMEDY_IN_FLIGHT, (uint32_t)first, (uint32_t)n, before, h->sel_bits,
                      h->sel_group, h->sel_acc));
    if (m) {
      ScanParams sc{};
      sc.group_count = h->sel_group;
      sc.group_prefix = h->sel_prefix;
      sc.acc = h->sel_acc;
      sc.n_groups = n_groups;
      sc.cap = 0xFFFFFFFFu;
      AM_CUDA(h, cudaMemsetAsync(h->sel_list, 0, m * 4, h->stream));
      AM_CUDA(h, launch(h, scan_groups_kernel, 1, 1024, h->stream, sc));
      AM_CUDA(h, launch(h, list_changes_kernel, n_groups, kGroupWords, h->stream, h->sel_bits,
                        (const uint32_t*)h->sel_prefix, h->sel_list));
      AM_CUDA(h, h->dev_in.reserve(m * 8));
      AM_CUDA(h, launch_values(h, state, first, h->sel_list, m, (int64_t*)h->dev_in.p));
    }
    // pin_in: the accumulators, m values, m list entries
    AM_CUDA(h, h->pin_in.reserve(16 + m * 12));
    char* p = (char*)h->pin_in.p;
    AM_CUDA(h, cudaMemcpyAsync(p, h->sel_acc, 16, cudaMemcpyDeviceToHost, h->stream));
    if (m) {
      AM_CUDA(h, cudaMemcpyAsync(p + 16, h->dev_in.p, m * 8, cudaMemcpyDeviceToHost, h->stream));
      AM_CUDA(h, cudaMemcpyAsync(p + 16 + m * 8, h->sel_list, m * 4, cudaMemcpyDeviceToHost, h->stream));
    }
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    const unsigned long long* acc = (const unsigned long long*)p;
    const uint64_t nm = acc[1];
    *n_match = nm;
    if (nm) *oldest = (int64_t)(acc[0] ^ (1ull << 63));
    const uint64_t k = std::min(cap, nm);
    const int64_t* vals = (const int64_t*)(p + 16);
    const uint32_t* list = (const uint32_t*)(p + 16 + m * 8);
    for (uint64_t j = 0; j < k; ++j) {
      idx[j] = h->shard_base + first + list[j];
      value[j] = vals[j];
    }
    return nm > cap ? AM_E_NOSPACE : AM_OK;
  });
}

// One of the last tick's two timed-out lists, entries [offset, ...) as global indices: the health-check runs, or the
// remedy runs with their start.
static int timed_out_impl(am_sweep_t* h, uint64_t offset, uint64_t* idx, int64_t* since, uint64_t cap, uint64_t* n_out,
                          bool remedy) {
  if (!h || (cap && (!idx || !since))) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (h->to_ran && !h->to_fetched) {  // the device list of the last tick, waited for (it may be on a caller stream)
    int rc = set_stream(h, h->stream);
    uint32_t m = 0;
    if (rc == AM_OK) rc = read_back(h, &m, h->to_count, 4);
    if (rc != AM_OK) return rc;
    std::vector<uint32_t> li(m);
    std::vector<int64_t> ls(m);
    if (m) {
      AM_CUDA(h, cudaMemcpy(li.data(), h->to_idx, m * 4ull, cudaMemcpyDeviceToHost));
      AM_CUDA(h, cudaMemcpy(ls.data(), h->to_since, m * 8ull, cudaMemcpyDeviceToHost));
    }
    h->to_host.clear();
    h->rto_host.clear();
    for (uint32_t k = 0; k < m; ++k)
      (is_remedy_run(ls[k]) ? h->rto_host : h->to_host).push_back({li[k], run_start(ls[k])});
    std::sort(h->to_host.begin(), h->to_host.end());  // (appended one segment at a time, in no particular order)
    std::sort(h->rto_host.begin(), h->rto_host.end());
    h->to_fetched = true;
  }
  const std::vector<std::pair<uint32_t, int64_t>>& list = remedy ? h->rto_host : h->to_host;
  uint64_t ncopy;
  const int page = list_page(h->to_ran ? list.size() : 0, offset, cap, n_out, &ncopy);
  if (page == AM_E_RANGE) return page;
  for (uint64_t k = 0; k < ncopy; ++k) {
    idx[k] = h->shard_base + list[offset + k].first;
    since[k] = list[offset + k].second;
  }
  return page;
}

// list_page over the last tick's change list (empty unless `listed`); its length is fetched once per tick.
static int change_page(am_sweep_t* h, bool listed, uint64_t offset, uint64_t cap, uint64_t* n_out, uint64_t* ncopy) {
  if (listed && !h->chg_fetched) {
    const int rc = read_back(h, &h->chg_n, h->chg_acc + 1, 8);
    if (rc != AM_OK) return rc;
    h->chg_fetched = true;
  }
  return list_page(listed ? h->chg_n : 0, offset, cap, n_out, ncopy);
}

// The bytes gather_cols fills for n slots: each requested column of `cols` (may be NULL), 8-B aligned.
static size_t gather_bytes(uint64_t n, const am_record_cols_t* cols) {
  size_t bytes = 0;
  for (int k = 0; k < 16; ++k)
    if (cols && *cols_member(cols, k)) bytes += (n * kColElem[k] + 7) / 8 * 8;
  return bytes;
}

// The requested columns of `cols` (may be NULL) at the n slots d_idx[0..n) (device memory), into the caller's arrays:
// gathered column by column into dev_in, copied to pin_in (both at least gather_bytes(n, cols) already, and what the
// caller keeps there lies past that), one synchronisation, then scattered.
static int gather_cols(am_sweep_t* h, const uint32_t* d_idx, uint64_t n, am_record_cols_t* cols) {
  GatherCols gc{};
  size_t at[16], bytes = 0;
  unsigned nc = 0;
  for (int k = 0; k < 16; ++k) {
    if (!cols || !*cols_member(cols, k)) continue;
    at[nc] = bytes;
    gc.src[nc] = *col_slot(h->cols, k);
    gc.dst[nc] = (char*)h->dev_in.p + bytes;
    gc.elem[nc] = (uint32_t)kColElem[k];
    bytes += (n * kColElem[k] + 7) / 8 * 8;
    ++nc;
  }
  if (nc) {
    AM_CUDA(h, launch(h, gather_columns_kernel, dim3((unsigned)((n + 255) / 256), nc), 256, h->stream, gc, d_idx,
                      (uint32_t)n));
    AM_CUDA(h, cudaMemcpyAsync(h->pin_in.p, h->dev_in.p, bytes, cudaMemcpyDeviceToHost, h->stream));
  }
  AM_CUDA(h, cudaStreamSynchronize(h->stream));
  for (int k = 0, c = 0; k < 16; ++k)
    if (cols && *cols_member(cols, k)) memcpy(*cols_member(cols, k), (const char*)h->pin_in.p + at[c++], n * kColElem[k]);
  return AM_OK;
}

int am_sweep_last_timed_out(am_sweep_t* h, uint64_t offset, uint64_t* idx, int64_t* since, uint64_t cap, uint64_t* n_out) {
  return timed_out_impl(h, offset, idx, since, cap, n_out, false);
}

int am_sweep_last_remedy_timed_out(am_sweep_t* h, uint64_t offset, uint64_t* idx, int64_t* started, uint64_t cap,
                                   uint64_t* n_out) {
  return timed_out_impl(h, offset, idx, started, cap, n_out, true);
}

int am_sweep_last_changes(am_sweep_t* h, uint64_t offset, uint64_t* idx, am_record_cols_t* cols, uint64_t cap,
                          uint64_t* n_out) {
  if (!h || (cap && !idx)) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->track) {
    h->last_error = "am_sweep_last_changes while tracking is off";
    return AM_E_INVAL;
  }
  int rc = set_stream(h, h->stream);  // (after the last tick, on whatever stream it ran; staged calls are not drained)
  if (rc != AM_OK) return rc;
  uint64_t ncopy;
  const int page = change_page(h, h->chg_listed, offset, cap, n_out, &ncopy);
  if (page != AM_OK && page != AM_E_NOSPACE) return page;
  if (ncopy) {
    // pin_in / dev_in: the requested columns, then (pin_in only) the list's entries
    const size_t at = gather_bytes(ncopy, cols);
    AM_CUDA(h, h->pin_in.reserve(at + ncopy * 4));
    AM_CUDA(h, h->dev_in.reserve(at));
    const uint32_t* d_idx = h->chg_list + offset;
    AM_CUDA(h, cudaMemcpyAsync((char*)h->pin_in.p + at, d_idx, ncopy * 4, cudaMemcpyDeviceToHost, h->stream));
    rc = gather_cols(h, d_idx, ncopy, cols);  // (synchronises)
    if (rc != AM_OK) return rc;
    const uint32_t* li = (const uint32_t*)((const char*)h->pin_in.p + at);
    for (uint64_t k = 0; k < ncopy; ++k) idx[k] = h->shard_base + li[k];
  }
  return page;
}

int am_sweep_last_change_details(am_sweep_t* h, uint64_t offset, uint64_t* idx, am_change_detail_t* out, uint64_t cap,
                                 uint64_t* n_out) {
  if (!h || (cap && (!idx || !out))) return AM_E_INVAL;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  if (!h->details) {
    h->last_error = "am_sweep_last_change_details while change details are off";
    return AM_E_INVAL;
  }
  int rc = set_stream(h, h->stream);  // (after the last tick, on whatever stream it ran; staged calls are not drained)
  if (rc != AM_OK) return rc;
  uint64_t ncopy;
  const int page = change_page(h, h->chg_listed && h->det_listed, offset, cap, n_out, &ncopy);
  if (page != AM_OK && page != AM_E_NOSPACE) return page;
  if (ncopy) {
    // pin_in / dev_in: the details, then the list's entries
    const size_t at = ncopy * sizeof(am_change_detail_t), bytes = at + ncopy * 4;
    AM_CUDA(h, h->pin_in.reserve(bytes));
    AM_CUDA(h, h->dev_in.reserve(bytes));
    const uint32_t* d_idx = h->chg_list + offset;
    AM_CUDA(h, launch(h, gather_details_kernel, (unsigned)((ncopy + 255) / 256), 256, h->stream, d_idx, (uint32_t)ncopy,
                      (const uint8_t*)h->det_e_applied + offset, (const int64_t*)h->det_e_start + offset,
                      h->set[h->chg_parity].out, h->chg_closed, h->chg_T, (am_change_detail_t*)h->dev_in.p));
    AM_CUDA(h, cudaMemcpyAsync(h->pin_in.p, h->dev_in.p, at, cudaMemcpyDeviceToHost, h->stream));
    AM_CUDA(h, cudaMemcpyAsync((char*)h->pin_in.p + at, d_idx, ncopy * 4, cudaMemcpyDeviceToHost, h->stream));
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    memcpy(out, h->pin_in.p, at);
    const uint32_t* li = (const uint32_t*)((const char*)h->pin_in.p + at);
    for (uint64_t k = 0; k < ncopy; ++k) idx[k] = h->shard_base + li[k];
  }
  return page;
}

// (tick guard held, staged events drained, h->stream ordered)
static int read_impl(am_sweep_t* h, uint64_t first, uint64_t n, const uint64_t* idx, am_record_cols_t* out) {
  int rc = check_slots(h, first, n, idx);
  if (rc != AM_OK) return rc;
  if (!idx) {
    for (int k = 0; k < 16; ++k) {
      void* dst = *cols_member(out, k);
      if (!dst) continue;
      AM_CUDA(h, cudaMemcpyAsync(dst, (char*)*col_slot(h->cols, k) + first * kColElem[k], n * kColElem[k],
                                 cudaMemcpyDeviceToHost, h->stream));
    }
    AM_CUDA(h, cudaStreamSynchronize(h->stream));
    return AM_OK;
  }
  const uint32_t* d_idx;
  rc = stage_indices(h, gather_bytes(n, out), n, idx, &d_idx);
  return rc != AM_OK ? rc : gather_cols(h, d_idx, n, out);
}

}  // extern "C"

// ---- checkpoints (DESIGN.md "Checkpoint format") ----------------------------------------------------------------------
namespace {

constexpr uint64_t kCkMagic = 0x54504B4357534D41ull;  // "AMSWCKPT"
constexpr uint64_t kCkHeader = 128;
constexpr uint32_t kCkAllSwitches =
    AM_CKPT_HOLD | AM_CKPT_REMEDY | AM_CKPT_TRACK | AM_CKPT_DETAILS | AM_CKPT_TIMEOUTS | AM_CKPT_ADMISSION;
constexpr size_t kCkChunk = 32u << 20;  // bytes per pinned chunk of a restore's upload

constexpr uint64_t kCkdMagic = 0x4C444B4357534D41ull;  // "AMSWCKDL"

// The header of a full blob and of a delta.  Words 10..13 are a delta's link; a full blob leaves them zero.  Word 14 is
// a packed blob's length once decoded (version 2; zero in version 1).
struct CkptHeader {
  uint64_t magic;
  uint32_t version, switches;
  uint64_t bytes, checksum, first_global, n, swept_end;
  int64_t prev_tick;
  uint64_t seed;
  uint32_t n_zones, reserved32;
  uint64_t n_changed, seq;
  int64_t parent_prev_tick;
  uint64_t parent_checksum;
  uint64_t raw_bytes;
  uint64_t reserved;
};
static_assert(sizeof(CkptHeader) == kCkHeader && kCkHeader == kCkHeaderBytes, "checkpoint header: 16 words");

// A blob's layout: the version-1 sections' offsets and end; where its zone table starts (the sections' end in version
// 1) and, packed, its blocks and the payload's bytes.
struct CkptLayout {
  uint64_t off[kCkSections] = {};
  uint64_t sections_end = kCkHeader;
  uint64_t zones_at = kCkHeader;
  uint64_t blocks = 0, payload = 0;
};

// The sections a blob of n slots with `switches` has, in order, each at an 8-B aligned offset from `start` on (a
// delta of n slots: ckd_start(n), after the offset section).
CkptLayout ckpt_layout(uint64_t n, uint32_t switches, uint64_t start = kCkHeader) {
  CkptLayout L;
  L.sections_end = L.zones_at = ck_layout(n, switches, start, L.off);
  return L;
}

uint64_t ckpt_zone_entry_bytes(size_t name_len) { return 8 + (name_len + 7) / 8 * 8; }

// Zeroes the bytes between each section's last element and the next 8-B boundary in the host copy `p` of a blob with
// n slots per section (layout L).  The staging area they are copied from keeps whatever an earlier blob with another
// layout left there, and blobs of one state must be equal byte for byte.
void ckpt_zero_padding(char* p, const CkptLayout& L, uint64_t n) {
  for (int s = 0; s < kCkSections; ++s) {
    if (!L.off[s]) continue;
    const uint64_t used = s == kCkSecChanged ? (n + 31) / 32 * 4 : n * ck_elem(s);
    memset(p + L.off[s] + used, 0, (used + 7) / 8 * 8 - used);
  }
}

// The checksum's terms of `len` bytes of words at `w`, which stand at byte `at` of the version-1 blob (the header, whose
// checksum word counts as 0, and the zone table).
uint64_t ckpt_host_sum(const void* w, uint64_t at, uint64_t len) {
  uint64_t s = 0;
  for (uint64_t o = 0; o < len; o += 8) {
    uint64_t v;
    memcpy(&v, (const char*)w + o, 8);
    if (at + o == offsetof(CkptHeader, checksum)) v = 0;
    s += ckpt_mix((at + o) * 8, v);
  }
  return s;
}

// The header of the version-1 blob a packed one decodes to: the checksum covers that one.
CkptHeader ckpt_v1_header(const CkptHeader& hd) {
  CkptHeader v = hd;
  if (v.version == AM_CHECKPOINT_VERSION_PACKED) {
    v.version = AM_CHECKPOINT_VERSION;
    v.bytes = hd.raw_bytes;
    v.raw_bytes = 0;
  }
  return v;
}

// The sections a packed blob of layout L (m elements per section; a delta's offsets first) encodes, at `blob` (the
// version-1 blob's byte 0) and `offs`; NULL for the geometry alone.
CkpSecs ckp_secs(const CkptLayout& L, uint64_t m, bool delta, char* blob, uint32_t* offs) {
  CkpSecs S{};
  uint64_t blk = 0;
  auto add = [&](char* p, uint64_t cnt, uint32_t esize, int64_t none) {
    S.p[S.n] = p;
    S.cnt[S.n] = cnt;
    S.esize[S.n] = esize;
    S.none[S.n] = none;
    S.blk0[S.n++] = blk;
    blk += (cnt + kCkpBlock - 1) / kCkpBlock;
  };
  if (delta) add((char*)offs, m, 4, 0);
  for (int q = 0; q < kCkSections; ++q) {
    if (!L.off[q]) continue;
    const bool bits = q == kCkSecChanged;
    add(blob ? blob + L.off[q] : nullptr, bits ? (m + 31) / 32 : m, bits ? 4 : ck_elem(q),
        q == kCkSecSince || q == kCkSecDetStart || q == kCkSecWait ? INT64_MIN
        : q == kCkSecDeadline                                      ? INT64_MAX
                                                                   : 0);
  }
  S.blk0[S.n] = blk;
  return S;
}

struct CkptZone {
  uint32_t id;
  std::string name;
};

// A full blob's or, with `delta`, a delta's header, layout and zone table (from the end of the sections to `bytes`),
// checked for consistency (not the checksum: that is a device pass).
int ckpt_parse(const void* buf, uint64_t len, bool delta, CkptHeader* hd, CkptLayout* L,
               std::vector<CkptZone>* zones) {
  if (!buf || len < kCkHeader) return AM_E_INVAL;
  memcpy(hd, buf, kCkHeader);
  const bool packed = hd->version == AM_CHECKPOINT_VERSION_PACKED;
  if (hd->magic != (delta ? kCkdMagic : kCkMagic) || (hd->version != AM_CHECKPOINT_VERSION && !packed))
    return AM_E_INVAL;
  if (delta && (hd->n_changed > hd->n || hd->seq == 0)) return AM_E_INVAL;
  if ((hd->switches & ~kCkAllSwitches) || ((hd->switches & AM_CKPT_REMEDY) && !(hd->switches & AM_CKPT_HOLD)) ||
      ((hd->switches & AM_CKPT_DETAILS) && !(hd->switches & AM_CKPT_TRACK)) ||
      ((hd->switches & AM_CKPT_ADMISSION) && !(hd->switches & AM_CKPT_HOLD)))
    return AM_E_INVAL;
  if (hd->bytes > len || hd->bytes % 8 || hd->n > 0xFFFFFFFFull || hd->first_global + hd->n < hd->first_global ||
      hd->swept_end < hd->first_global || hd->swept_end > hd->first_global + hd->n || hd->n_zones > 255)
    return AM_E_INVAL;
  const uint64_t m = delta ? hd->n_changed : hd->n;
  *L = delta ? ckpt_layout(m, hd->switches, ckd_start(m)) : ckpt_layout(hd->n, hd->switches);
  const char* p = (const char*)buf;
  if (packed) {  // the directory, then the payload up to the end of the last block's, then the zone table
    const CkpSecs S = ckp_secs(*L, m, delta, nullptr, nullptr);
    L->blocks = S.blk0[S.n];
    const uint64_t dir_end = kCkHeader + L->blocks * sizeof(CkpEntry);
    if (L->blocks > hd->bytes / sizeof(CkpEntry) || dir_end > hd->bytes) return AM_E_INVAL;
    if (L->blocks) {
      CkpEntry e;
      memcpy(&e, p + dir_end - sizeof(CkpEntry), sizeof e);
      const int s = S.n - 1;  // (the last section has the last block: m > 0)
      const uint64_t cnt = S.cnt[s] - (L->blocks - 1 - S.blk0[s]) * kCkpBlock;
      if (!ckp_entry_ok(e, cnt, S.esize[s]) || e.off > hd->bytes) return AM_E_INVAL;
      L->payload = e.off + ckp_bytes(e.mode, e.width, e.aux, cnt, S.esize[s]);
    }
    // (no block is larger than its elements verbatim: the encoder falls back to RAW)
    if (L->payload > L->sections_end - kCkHeader || dir_end + L->payload > hd->bytes) return AM_E_INVAL;
    L->zones_at = dir_end + L->payload;
  }
  uint64_t at = L->zones_at;  // (past `bytes` when a delta's n_changed is out of range: refused below)
  bool seen[256] = {};
  zones->clear();
  for (uint32_t k = 0; k < hd->n_zones; ++k) {
    if (at + 8 > hd->bytes) return AM_E_INVAL;
    uint32_t id, nl;
    memcpy(&id, p + at, 4);
    memcpy(&nl, p + at + 4, 4);
    if (id < 1 || id > 255 || seen[id] || nl < 1 || nl > 255 || at + ckpt_zone_entry_bytes(nl) > hd->bytes)
      return AM_E_INVAL;
    seen[id] = true;
    zones->push_back({id, std::string(p + at + 8, nl)});
    at += ckpt_zone_entry_bytes(nl);
  }
  if (packed && hd->raw_bytes != L->sections_end + (hd->bytes - L->zones_at)) return AM_E_INVAL;
  return at == hd->bytes ? AM_OK : AM_E_INVAL;
}

// The zones a pass marked (8 words of marks, one bit per id) with their names.  AM_E_DEVICE: an id that is not
// registered (upserts and loads refuse those).
int ckpt_marked_zones(am_sweep* h, const uint32_t* marks, const char* who, std::vector<CkptZone>* zones) {
  zones->clear();
  for (uint32_t id = 1; id < 256; ++id) {
    if (!((marks[id >> 5] >> (id & 31)) & 1u)) continue;
    std::string name;
    if (!amsweep_tz::name_of((int32_t)id, &name)) {
      h->last_error = std::string(who) + ": a record carries a zone id that is not registered";
      return AM_E_DEVICE;
    }
    zones->push_back({id, name});
  }
  return AM_OK;
}
// ... written as a zone table at p + at; returns its end
uint64_t ckpt_put_zones(char* p, uint64_t at, const std::vector<CkptZone>& zones) {
  for (const CkptZone& z : zones) {
    const uint32_t nl = (uint32_t)z.name.size();
    memset(p + at, 0, ckpt_zone_entry_bytes(nl));
    memcpy(p + at, &z.id, 4);
    memcpy(p + at + 4, &nl, 4);
    memcpy(p + at + 8, z.name.data(), nl);
    at += ckpt_zone_entry_bytes(nl);
  }
  return at;
}
// A blob's zone table resolved to this process's ids with am_tz_lookup (id 0 stays 0).
int ckpt_zone_lut(am_sweep* h, const std::vector<CkptZone>& zones, const char* who, ZoneLut* lut) {
  *lut = ZoneLut{};
  for (const CkptZone& z : zones) {
    int32_t id = 0;
    const int rc = am_tz_lookup(z.name.data(), z.name.size(), &id);
    if (rc != AM_OK) {
      h->last_error =
          std::string(who) + ": time zone " + z.name + (rc == AM_E_PARSE ? " is unknown here" : " does not fit the registry");
      return rc;
    }
    lut->id[z.id] = (uint8_t)id;
  }
  return AM_OK;
}

uint32_t ckpt_switches(const am_sweep* h) {
  return (h->hold ? AM_CKPT_HOLD : 0u) | (h->remedy ? AM_CKPT_REMEDY : 0u) | (h->track ? AM_CKPT_TRACK : 0u) |
         (h->details ? AM_CKPT_DETAILS : 0u) | (h->wf_timeout ? AM_CKPT_TIMEOUTS : 0u) |
         (admission_on(h) ? AM_CKPT_ADMISSION : 0u);
}

// The checkpoint state of a handle, at the first checkpoint or restore (ck_mu held).
int ckpt_alloc(am_sweep* h) {
  AM_CUDA(h, cudaSetDevice(h->device));
  if (h->ck_dev) return AM_OK;
  AM_CUDA(h, new_stream(h, &h->ck_stream));
  AM_CUDA(h, new_event(h, &h->ck_ev));
  for (int k = 0; k < 2; ++k) {
    AM_CUDA(h, new_event(h, &h->ck_pin_ev[k]));
    AM_CUDA(h, host_array(h, &h->ck_pin[k], kCkChunk));
  }
  AM_CUDA(h, host_array(h, &h->ck_meta_h, 5 * 8));
  AM_CUDA(h, dev_array(h, &h->ck_meta, 5 * 8, h->ck_stream, false));
  const uint64_t blob = ckpt_layout(h->cap_padded, kCkAllSwitches).sections_end;
  AM_CUDA(h, dev_array(h, &h->ck_dev, blob, h->ck_stream, false));  // (the last)
  return AM_OK;
}

CkptState ckpt_state(am_sweep* h) {
  CkptState s{};
  for (int k = 0; k < 16; ++k) s.col[k] = *col_slot(h->cols, k);
  if (h->wf_timeout) {
    s.wf_timeout = h->wf_timeout;
    s.deadline = h->deadline;
    s.seg_deadline = h->seg_deadline;
  }
  if (h->hold) s.since = h->since;
  if (h->track) s.changed = h->chg_bits;
  if (h->details) {
    s.det_applied = h->det_applied;
    s.det_start = h->det_start;
  }
  if (admission_on(h)) s.wait = h->adm_wait;
  return s;
}

// A blob of n elements per section (layout L) in the staging area: its sections from byte 128 of ck_dev on (a delta's
// offsets are in ckd_off).
CkptBlob ckpt_blob(const am_sweep* h, const CkptLayout& L, uint64_t n) {
  CkptBlob b{};
  b.p = h->ck_dev + kCkHeader - L.off[0];
  memcpy(b.off, L.off, sizeof b.off);
  b.n = n;
  return b;
}
// The chain's base image: the previous link's sections over the chain's n slots, in the root's layout.
CkptBlob ckd_base_blob(const am_sweep* h, uint64_t n, uint32_t switches) {
  CkptBlob b = ckpt_blob(h, ckpt_layout(n, switches), n);
  b.p = h->ckd_base;
  return b;
}

// The delta state of a handle (ck_mu held, after ckpt_alloc): the offsets and accumulators on both sides; the base
// image, the bitmap and the group arrays on a producer.
int ckd_alloc(am_sweep* h, bool producer) {
  if (!h->ckd_off) {
    AM_CUDA(h, dev_array(h, &h->ckd_acc, 4 * 8, h->ck_stream));
    AM_CUDA(h, host_array(h, &h->ckd_acc_h, 4 * 8));
    AM_CUDA(h, dev_array(h, &h->ckd_off, h->cap_padded * 4, h->ck_stream, false));  // (the last)
  }
  if (producer && !h->ckd_base) {
    const size_t ngroups = groups_of(h->cap_padded);
    AM_CUDA(h, dev_array(h, &h->ckd_bits, ngroups * kGroupWords * 4, h->ck_stream));
    AM_CUDA(h, dev_array(h, &h->ckd_group, ngroups * 4, h->ck_stream));
    AM_CUDA(h, dev_array(h, &h->ckd_prefix, (ngroups + 1) * 4, h->ck_stream, false));
    AM_CUDA(h, dev_array(h, &h->ckd_base, ckpt_layout(h->cap_padded, kCkAllSwitches).sections_end, h->ck_stream,
                         false));  // (the last)
  }
  AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));  // (the zeroed arrays are read on the handle's stream)
  return AM_OK;
}

// The packed staging area of a handle, at its first packed checkpoint or restore (ck_mu held, after ckpt_alloc).
// AM_E_UNSUPPORTED: a capacity whose payload would not fit the scan's u32 word counts.
int ckp_alloc(am_sweep* h) {
  if (h->ckp_dev) return AM_OK;
  const CkptLayout L = ckpt_layout(h->cap_padded, kCkAllSwitches, ckd_start(h->cap_padded));
  const CkpSecs S = ckp_secs(L, h->cap_padded, true, nullptr, nullptr);
  const uint64_t nb = S.blk0[S.n];
  const uint64_t payload = L.sections_end - kCkHeader;
  if (payload / 8 > 0xFFFFFFFFull) {
    h->last_error = "packed checkpoints: the capacity is too large for the encoder's 32-bit payload word counts";
    return AM_E_UNSUPPORTED;
  }
  AM_CUDA(h, dev_array(h, &h->ckp_words, nb * 4, h->ck_stream, false));
  AM_CUDA(h, dev_array(h, &h->ckp_prefix, (nb + 1) * 4, h->ck_stream, false));
  AM_CUDA(h, dev_array(h, &h->ckp_base, nb * 8, h->ck_stream, false));
  AM_CUDA(h, dev_array(h, &h->ckp_acc, 4 * 8, h->ck_stream));
  AM_CUDA(h, host_array(h, &h->ckp_acc_h, 4 * 8));
  AM_CUDA(h, dev_array(h, &h->ckp_dev, nb * sizeof(CkpEntry) + payload, h->ck_stream, false));  // (the last)
  AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
  return AM_OK;
}

// `bytes` at `src` (host) to `dst` (device) on the checkpoint stream, in chunks through the two pinned buffers (the
// host fills one while the other crosses).
int ckpt_upload(am_sweep* h, char* dst, const char* src, uint64_t bytes) {
  for (uint64_t off = 0, k = 0; off < bytes; off += kCkChunk, ++k) {
    const size_t m = (size_t)std::min<uint64_t>(kCkChunk, bytes - off);
    const int b = (int)(k & 1);
    if (h->ck_pin_pending[b]) AM_CUDA(h, cudaEventSynchronize(h->ck_pin_ev[b]));
    memcpy(h->ck_pin[b], src + off, m);
    AM_CUDA(h, cudaMemcpyAsync(dst + off, h->ck_pin[b], m, cudaMemcpyHostToDevice, h->ck_stream));
    AM_CUDA(h, cudaEventRecord(h->ck_pin_ev[b], h->ck_stream));
    h->ck_pin_pending[b] = true;
  }
  return AM_OK;
}

// A restore's refusal after the checksum (tick guard held): switches, the timeout state aside, that differ from the
// handle's.
int ckpt_restore_switches(am_sweep* h, uint32_t switches, const char* who) {
  if ((switches & ~AM_CKPT_TIMEOUTS) != (ckpt_switches(h) & ~AM_CKPT_TIMEOUTS)) {
    h->last_error = std::string(who) + ": set the handle's switches to the blob's first (am_checkpoint_info)";
    return AM_E_INVAL;
  }
  return AM_OK;
}

// A blob a restore has checked and staged: its header, its layout, its zone ids here, and its first slot in the handle.
struct CkptRestore {
  bool delta;
  CkptHeader hd;
  CkptLayout L;
  ZoneLut lut;
  uint64_t first;
  uint64_t m;  // elements per section: n, or a delta's n_changed
};

// A restore's steps before anything of the handle changes (ck_mu held): the blob `buf` (a delta with `delta`) parsed,
// its range checked against the shard and its zone table resolved; its sections (and a delta's offsets) up in chunks,
// then the device passes that verify the checksum (and that the offsets ascend inside the range) and the zone ids its
// records use.
int ckpt_restore_check(am_sweep* h, const void* buf, uint64_t len, bool delta, CkptRestore* r) {
  const char* who = delta ? "am_sweep_restore_delta" : "am_sweep_restore";
  const std::string what = delta ? "delta" : "blob";
  const CkptHeader& hd = r->hd;
  std::vector<CkptZone> zones;
  r->delta = delta;
  int rc = ckpt_parse(buf, len, delta, &r->hd, &r->L, &zones);
  if (rc != AM_OK) {
    h->last_error = std::string(who) + ": not a " + (delta ? "delta" : "checkpoint") +
                    " of this format version, or truncated";
    return rc;
  }
  if (hd.first_global < h->shard_base || hd.first_global - h->shard_base + hd.n > h->capacity) {
    h->last_error = std::string(who) + ": the " + what + "'s slots are not all inside this shard";
    return AM_E_RANGE;
  }
  r->first = hd.first_global - h->shard_base;
  r->m = delta ? hd.n_changed : hd.n;
  rc = ckpt_zone_lut(h, zones, who, &r->lut);
  if (rc != AM_OK) return rc;
  rc = ckpt_alloc(h);
  if (rc == AM_OK && delta) rc = ckd_alloc(h, false);
  if (rc != AM_OK) return rc;
  const char* p = (const char*)buf;
  const uint64_t m = r->m, start = r->L.off[0];
  const bool packed = hd.version == AM_CHECKPOINT_VERSION_PACKED;
  if (packed) {  // the directory and payload up; the directory validated, then decoded into the version-1 places
    rc = ckp_alloc(h);
    if (rc == AM_OK) rc = ckpt_upload(h, h->ckp_dev, p + kCkHeader, r->L.zones_at - kCkHeader);
    if (rc != AM_OK) return rc;
    AM_CUDA(h, cudaMemsetAsync(h->ckp_acc, 0, 4 * 8, h->ck_stream));
    const CkpSecs S = ckp_secs(r->L, m, delta, ckpt_blob(h, r->L, m).p, h->ckd_off);
    const uint64_t nb = r->L.blocks;
    const CkpEntry* dir = (const CkpEntry*)h->ckp_dev;
    if (nb) {
      AM_CUDA(h, launch(h, ckp_validate_kernel, (unsigned)((nb + 255) / 256), 256, h->ck_stream, S, dir,
                        r->L.payload, (uint32_t*)(h->ckp_acc + 2)));
      AM_CUDA(h, launch(h, ckp_decode_kernel, (unsigned)nb, kCkpThreads, h->ck_stream, S, dir,
                        (const char*)(dir + nb), (uint32_t*)(h->ckp_acc + 2)));
    }
    AM_CUDA(h, cudaMemcpyAsync(h->ckp_acc_h, h->ckp_acc, 4 * 8, cudaMemcpyDeviceToHost, h->ck_stream));
  } else {
    if (delta) rc = ckpt_upload(h, (char*)h->ckd_off, p + kCkHeader, m * 4);
    if (rc == AM_OK) rc = ckpt_upload(h, h->ck_dev + kCkHeader, p + start, r->L.sections_end - start);
    if (rc != AM_OK) return rc;
  }
  AM_CUDA(h, cudaMemsetAsync(h->ck_meta, 0, 5 * 8, h->ck_stream));
  if (delta) AM_CUDA(h, cudaMemsetAsync(h->ckd_acc, 0, 4 * 8, h->ck_stream));
  if (m) {
    const unsigned grid = (unsigned)((m + 255) / 256);
    if (delta)
      AM_CUDA(h, launch(h, delta_offsets_verify_kernel, grid, 256, h->ck_stream, (const uint32_t*)h->ckd_off, m, hd.n,
                        h->ck_meta, (uint32_t*)(h->ckd_acc + 2)));
    AM_CUDA(h, launch(h, checkpoint_verify_kernel, grid, 256, h->ck_stream, ckpt_blob(h, r->L, m), h->ck_meta,
                      (uint32_t*)(h->ck_meta + 1)));
  }
  AM_CUDA(h, cudaMemcpyAsync(h->ck_meta_h, h->ck_meta, 5 * 8, cudaMemcpyDeviceToHost, h->ck_stream));
  if (delta) AM_CUDA(h, cudaMemcpyAsync(h->ckd_acc_h, h->ckd_acc, 4 * 8, cudaMemcpyDeviceToHost, h->ck_stream));
  AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
  h->ck_pin_pending[0] = h->ck_pin_pending[1] = false;
  if (packed && h->ckp_acc_h[2]) {
    h->last_error = std::string(who) + ": a packed block or its directory entry is malformed";
    return AM_E_INVAL;
  }
  const CkptHeader v1 = ckpt_v1_header(hd);
  const uint64_t sum = h->ck_meta_h[0] + ckpt_host_sum(&v1, 0, kCkHeader) +
                       ckpt_host_sum(p + r->L.zones_at, r->L.sections_end, hd.bytes - r->L.zones_at);
  if (sum != hd.checksum) {
    h->last_error = std::string(who) + ": checksum mismatch";
    return AM_E_INVAL;
  }
  if (delta && h->ckd_acc_h[2]) {
    h->last_error = std::string(who) + ": the slot offsets are not strictly ascending inside the range";
    return AM_E_INVAL;
  }
  const uint32_t* marks = (const uint32_t*)(h->ck_meta_h + 1);
  for (uint32_t id = 1; id < 256; ++id)
    if (((marks[id >> 5] >> (id & 31)) & 1u) && !r->lut.id[id]) {
      h->last_error = std::string(who) + ": a record names a zone the " + what + "'s table does not";
      return AM_E_INVAL;
    }
  return AM_OK;
}

// The rest of a restore once its entry point's own preconditions hold (tick guard held).  A restore is a call in the
// per-slot order: the calls staged before it are applied first, and it replaces them.  Then the timeout state the
// blob carries, the scatter and the planes of its slots (a full restore's rebuild_planes drops the due words, a
// delta's scatter keeps them exact), the high-water mark, the admission order, P and the seed; the previous tick's
// lists are not carried: empty until the next tick.
int ckpt_restore_apply(am_sweep* h, const CkptRestore& r) {
  const CkptHeader& hd = r.hd;
  int rc = begin_call(h);
  if (rc != AM_OK) return rc;
  if ((hd.switches & AM_CKPT_TIMEOUTS) && !h->wf_timeout) {
    rc = alloc_timeouts(h, h->stream);
    if (rc != AM_OK) return rc;
  }
  if (r.m && r.delta) {
    AM_CUDA(h, launch(h, delta_scatter_kernel, (unsigned)((r.m + 255) / 256), 256, h->stream, ckpt_state(h),
                      ckpt_blob(h, r.L, r.m), (const uint32_t*)h->ckd_off, r.first, r.lut, h->seg_dirty, due_kept(h),
                      h->due_epoch));
    AM_CUDA(h, launch(h, delta_planes_kernel, (unsigned)((r.m + kWarps - 1) / kWarps), kBlock, h->stream, h->cols,
                      h->planes, h->seg_dirty, (const uint32_t*)h->ckd_off, r.first, (uint32_t)r.m));
  } else if (r.m) {
    AM_CUDA(h, launch(h, checkpoint_scatter_kernel, (unsigned)((r.m + 255) / 256), 256, h->stream, ckpt_state(h),
                      ckpt_blob(h, r.L, r.m), r.first, r.lut));
    rc = rebuild_planes(h, r.first, r.m);
    if (rc != AM_OK) return rc;
  }
  AM_CUDA(h, cudaStreamSynchronize(h->stream));
  const uint64_t hwm = hd.swept_end - h->shard_base;
  if (hwm > h->n_records) set_hwm(h, hwm);
  if (admission_on(h)) {  // the admission order of every waiting slot of the handle, from the waits as they now stand
    rc = rebuild_admission_fifo(h);
    if (rc != AM_OK) return rc;
  }
  if (hd.prev_tick != INT64_MIN) {
    h->has_prev = true;
    h->prev_T = hd.prev_tick;
  }
  h->seed = hd.seed;
  h->host_n = 0;
  h->to_ran = h->to_fetched = false;
  h->chg_listed = h->chg_fetched = false;
  return AM_OK;
}

// The header words every blob of the slots [first, first + n) carries: the handle's switches, P and seed (tick guard
// held).  The producer fills in the rest at its seal.
CkptHeader ckpt_header(const am_sweep* h, uint64_t magic, uint64_t first, uint64_t n) {
  CkptHeader hd{};
  hd.magic = magic;
  hd.version = AM_CHECKPOINT_VERSION;
  hd.switches = ckpt_switches(h);
  hd.first_global = h->shard_base + first;
  hd.n = n;
  hd.swept_end = h->shard_base + std::min(std::max(h->n_records, first), first + n);
  hd.prev_tick = h->has_prev ? h->prev_T : INT64_MIN;
  hd.seed = h->seed;
  return hd;
}

// The end of a producer, after its pass (ck_ev): the blob of the staging area's sections (n elements each, layout L;
// with `delta` the offsets in ckd_off first) and the zone table of the pass's marks (`zones`) into the caller's
// buffer `p`, with the header *hd and the checksum word; *len_out = the blob's length.  AM_E_NOSPACE (*len_out = the
// length) when cap is below it.  While the handle packs, the encode runs first on the checkpoint stream and the blob
// is packed (DESIGN.md "Packed format"); its checksum is that of the version-1 blob it decodes to.
int ckpt_seal(am_sweep* h, char* p, uint64_t cap, CkptHeader* hd, const CkptLayout& L, uint64_t n, bool delta,
              const std::vector<CkptZone>& zones, uint64_t* len_out) {
  uint64_t zone_bytes = 0;
  for (const CkptZone& z : zones) zone_bytes += ckpt_zone_entry_bytes(z.name.size());
  hd->n_zones = (uint32_t)zones.size();
  hd->bytes = L.sections_end + zone_bytes;
  AM_CUDA(h, cudaStreamWaitEvent(h->ck_stream, h->ck_ev, 0));
  if (h->ck_packing) {
    int rc = ckp_alloc(h);
    if (rc != AM_OK) return rc;
    const CkpSecs S = ckp_secs(L, n, delta, ckpt_blob(h, L, n).p, h->ckd_off);
    const uint64_t nb = S.blk0[S.n];
    CkpEntry* dir = (CkpEntry*)h->ckp_dev;
    uint64_t payload = 0;
    if (nb) {  // sizes, their scan into word offsets, the payloads; one synchronisation for the packed length
      AM_CUDA(h, launch(h, ckp_size_kernel, (unsigned)nb, kCkpThreads, h->ck_stream, S, dir, h->ckp_words,
                        h->ckp_base));
      ScanParams sc{};
      sc.group_count = h->ckp_words;
      sc.group_prefix = h->ckp_prefix;
      sc.acc = h->ckp_acc;
      sc.n_groups = (uint32_t)nb;
      sc.cap = 0xFFFFFFFFu;
      AM_CUDA(h, launch(h, scan_groups_kernel, 1, 1024, h->ck_stream, sc));
      AM_CUDA(h, launch(h, ckp_write_kernel, (unsigned)nb, kCkpThreads, h->ck_stream, S, dir,
                        (const uint32_t*)h->ckp_prefix, (const int64_t*)h->ckp_base, (char*)(dir + nb)));
      AM_CUDA(h, cudaMemcpyAsync(h->ckp_acc_h, h->ckp_acc, 4 * 8, cudaMemcpyDeviceToHost, h->ck_stream));
      AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
      payload = h->ckp_acc_h[1] * 8;
    }
    const uint64_t at = kCkHeader + nb * sizeof(CkpEntry) + payload;
    if (cap < at + zone_bytes) {
      *len_out = at + zone_bytes;
      return AM_E_NOSPACE;
    }
    ckpt_put_zones(p, at, zones);
    hd->checksum = h->ck_meta_h[0] + ckpt_host_sum(hd, 0, kCkHeader) + ckpt_host_sum(p + at, L.sections_end, zone_bytes);
    hd->version = AM_CHECKPOINT_VERSION_PACKED;
    hd->raw_bytes = hd->bytes;
    hd->bytes = at + zone_bytes;
    memcpy(p, hd, kCkHeader);
    if (at > kCkHeader)
      AM_CUDA(h, cudaMemcpyAsync(p + kCkHeader, h->ckp_dev, at - kCkHeader, cudaMemcpyDeviceToHost, h->ck_stream));
    AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
    *len_out = hd->bytes;
    return AM_OK;
  }
  if (cap < hd->bytes) {  // (a full blob's room was checked before its pass, for every registered zone)
    *len_out = hd->bytes;
    return AM_E_NOSPACE;
  }
  ckpt_put_zones(p, L.sections_end, zones);
  memcpy(p, hd, kCkHeader);
  if (L.sections_end > L.off[0])  // (the sections start at L.off[0]: the header's end, or a delta's offsets' end)
    AM_CUDA(h, cudaMemcpyAsync(p + L.off[0], h->ck_dev + kCkHeader, L.sections_end - L.off[0], cudaMemcpyDeviceToHost,
                               h->ck_stream));
  if (delta && n)  // the offset section (its checksum terms are the pack's)
    AM_CUDA(h, cudaMemcpyAsync(p + kCkHeader, h->ckd_off, n * 4, cudaMemcpyDeviceToHost, h->ck_stream));
  AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
  ckpt_zero_padding(p, L, n);
  if (delta) memset(p + kCkHeader + n * 4, 0, L.off[0] - kCkHeader - n * 4);
  hd->checksum = h->ck_meta_h[0] + ckpt_host_sum(p, 0, kCkHeader) +
                 ckpt_host_sum(p + L.sections_end, L.sections_end, hd->bytes - L.sections_end);
  memcpy(p + offsetof(CkptHeader, checksum), &hd->checksum, 8);
  *len_out = hd->bytes;
  return AM_OK;
}

// A full checkpoint (am_sweep_checkpoint, ck_mu held); *hd and *L = its header and layout.
int checkpoint_locked(am_sweep* h, uint64_t first, uint64_t n, void* buf, uint64_t cap, uint64_t* len_out,
                      CkptHeader* hd, CkptLayout* L) {
  {  // the pass, with the tick guard held: the drain, then one kernel over the range on the handle's stream
    TickGuard g(h);
    if (!g.ok) return AM_E_BUSY;
    int rc = begin_call(h);  // (first: the drain may allocate the timeout state, a section of the blob)
    if (rc != AM_OK) return rc;
    *hd = ckpt_header(h, kCkMagic, first, n);
    *L = ckpt_layout(n, hd->switches);
    uint64_t bound = L->sections_end;  // (room for the names of every registered zone; a packed blob's after its encode)
    std::string name;
    for (int32_t id = 1; amsweep_tz::name_of(id, &name); ++id) bound += ckpt_zone_entry_bytes(name.size());
    if (cap < bound && !h->ck_packing) {
      *len_out = bound;
      return AM_E_NOSPACE;
    }
    rc = ckpt_alloc(h);
    if (rc != AM_OK) return rc;
    AM_CUDA(h, cudaMemsetAsync(h->ck_meta, 0, 5 * 8, h->stream));
    if (n)
      AM_CUDA(h, launch(h, checkpoint_pack_kernel, (unsigned)((n + 255) / 256), 256, h->stream, ckpt_state(h),
                        ckpt_blob(h, *L, n), first, h->ck_meta, (uint32_t*)(h->ck_meta + 1)));
    AM_CUDA(h, cudaMemcpyAsync(h->ck_meta_h, h->ck_meta, 5 * 8, cudaMemcpyDeviceToHost, h->stream));
    AM_CUDA(h, cudaEventRecord(h->ck_ev, h->stream));
  }
  // Ticks may run from here on: the copy to the caller waits for the pass only, on the checkpoint stream.
  AM_CUDA(h, cudaEventSynchronize(h->ck_ev));
  std::vector<CkptZone> zones;
  const int rc = ckpt_marked_zones(h, (const uint32_t*)(h->ck_meta_h + 1), "am_sweep_checkpoint", &zones);
  if (rc != AM_OK) return rc;
  return ckpt_seal(h, (char*)buf, cap, hd, *L, n, false, zones, len_out);
}

// A restored full blob starts the handle's link entry for its range, replacing every entry that overlaps it.
void ckpt_start_link(am_sweep* h, uint64_t first_global, uint64_t n, uint64_t checksum) {
  auto& v = h->links;
  v.erase(std::remove_if(v.begin(), v.end(),
                         [&](const CkptLink& e) {
                           return e.first_global < first_global + n && first_global < e.first_global + e.n;
                         }),
          v.end());
  v.push_back({first_global, n, checksum, h->ticks});
}


}  // namespace

extern "C" {

int am_sweep_checkpoint(am_sweep_t* h, uint64_t first, uint64_t n, void* buf, uint64_t cap, uint64_t* len_out) {
  if (!h || !len_out || (cap && !buf)) return AM_E_INVAL;
  if (first + n > h->capacity || first + n < first) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  CkptHeader hd;
  CkptLayout L;
  return checkpoint_locked(h, first, n, buf, cap, len_out, &hd, &L);
}

int am_sweep_set_checkpoint_packing(am_sweep_t* h, int on) {
  if (!h) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  h->ck_packing = on != 0;
  return AM_OK;
}

int am_checkpoint_info(const void* buf, uint64_t len, am_checkpoint_info_t* info) {
  if (!info) return AM_E_INVAL;
  CkptHeader hd;
  CkptLayout L;
  std::vector<CkptZone> zones;
  const int rc = ckpt_parse(buf, len, false, &hd, &L, &zones);
  if (rc != AM_OK) return rc;
  *info = am_checkpoint_info_t{};
  info->first_global = hd.first_global;
  info->n = hd.n;
  info->swept_end = hd.swept_end;
  info->prev_tick = hd.prev_tick;
  info->seed = hd.seed;
  info->switches = hd.switches;
  info->n_zones = hd.n_zones;
  info->version = hd.version;
  info->bytes = hd.bytes;
  return AM_OK;
}

int am_sweep_restore(am_sweep_t* h, const void* buf, uint64_t len) {
  if (!h || !buf) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  CkptRestore r;
  int rc = ckpt_restore_check(h, buf, len, false, &r);
  if (rc != AM_OK) return rc;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  rc = ckpt_restore_switches(h, r.hd.switches, "am_sweep_restore");
  if (rc != AM_OK) return rc;
  if (h->has_prev && (r.hd.prev_tick == INT64_MIN || r.hd.prev_tick != h->prev_T)) {
    h->last_error = "am_sweep_restore: the handle's previous tick differs from the blob's";
    return AM_E_INVAL;
  }
  rc = ckpt_restore_apply(h, r);
  if (rc != AM_OK) return rc;
  ckpt_start_link(h, r.hd.first_global, r.hd.n, r.hd.checksum);
  return AM_OK;
}

int am_sweep_checkpoint_chain(am_sweep_t* h, uint64_t first, uint64_t n, void* buf, uint64_t cap, uint64_t* len_out) {
  if (!h || !len_out || (cap && !buf)) return AM_E_INVAL;
  if (first + n > h->capacity || first + n < first) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  int rc = ckpt_alloc(h);
  if (rc == AM_OK) rc = ckd_alloc(h, true);
  if (rc != AM_OK) return rc;
  CkptHeader hd;
  CkptLayout L;
  rc = checkpoint_locked(h, first, n, buf, cap, len_out, &hd, &L);
  if (rc != AM_OK) return rc;
  // the root's sections become the chain's base image (the staging area holds them until the next checkpoint)
  if (L.sections_end > kCkHeader)
    AM_CUDA(h, cudaMemcpyAsync(h->ckd_base + kCkHeader, h->ck_dev + kCkHeader, L.sections_end - kCkHeader,
                               cudaMemcpyDeviceToDevice, h->ck_stream));
  AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
  h->chain = true;
  h->chain_first = first;
  h->chain_n = n;
  h->chain_switches = hd.switches;
  h->chain_checksum = hd.checksum;
  h->chain_seq = 0;
  h->chain_prev_tick = hd.prev_tick;
  return AM_OK;
}

int am_sweep_checkpoint_delta(am_sweep_t* h, void* buf, uint64_t cap, uint64_t* len_out, uint64_t* n_changed) {
  if (!h || !len_out || !n_changed || (cap && !buf)) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  if (!h->chain) {
    h->last_error = "am_sweep_checkpoint_delta: the handle has no chain (am_sweep_checkpoint_chain)";
    return AM_E_INVAL;
  }
  const uint64_t first = h->chain_first, n = h->chain_n;
  CkptHeader hd;
  {  // the passes, with the tick guard held: the drain, then the diff, its compaction and the pack on the handle's stream
    TickGuard g(h);
    if (!g.ok) return AM_E_BUSY;
    const int rc = begin_call(h);
    if (rc != AM_OK) return rc;
    if (ckpt_switches(h) != h->chain_switches) {
      h->last_error = "am_sweep_checkpoint_delta: the switches differ from the chain root's: start a new chain";
      return AM_E_INVAL;
    }
    hd = ckpt_header(h, kCkdMagic, first, n);
    hd.seq = h->chain_seq + 1;
    hd.parent_prev_tick = h->chain_prev_tick;
    hd.parent_checksum = h->chain_checksum;
    AM_CUDA(h, cudaMemsetAsync(h->ck_meta, 0, 5 * 8, h->stream));
    if (n) {
      const unsigned grid = (unsigned)((n + 255) / 256);
      AM_CUDA(h, launch(h, delta_diff_kernel, grid, 256, h->stream, ckpt_state(h),
                        ckd_base_blob(h, n, hd.switches), first, h->ckd_bits, h->ckd_group));
      ScanParams sc{};
      sc.group_count = h->ckd_group;
      sc.group_prefix = h->ckd_prefix;
      sc.acc = h->ckd_acc;
      sc.n_groups = groups_of(n);
      sc.cap = 0xFFFFFFFFu;
      AM_CUDA(h, launch(h, scan_groups_kernel, 1, 1024, h->stream, sc));
      AM_CUDA(h, launch(h, list_changes_kernel, sc.n_groups, kGroupWords, h->stream, h->ckd_bits,
                        (const uint32_t*)h->ckd_prefix, h->ckd_off));
      AM_CUDA(h, launch(h, delta_pack_kernel, grid, 256, h->stream, ckpt_state(h), h->ck_dev, hd.switches,
                        (const uint32_t*)h->ckd_off, (const unsigned long long*)(h->ckd_acc + 1), first, h->ck_meta,
                        (uint32_t*)(h->ck_meta + 1)));
      AM_CUDA(h, cudaMemcpyAsync(h->ckd_acc_h, h->ckd_acc, 4 * 8, cudaMemcpyDeviceToHost, h->stream));
    }
    AM_CUDA(h, cudaMemcpyAsync(h->ck_meta_h, h->ck_meta, 5 * 8, cudaMemcpyDeviceToHost, h->stream));
    AM_CUDA(h, cudaEventRecord(h->ck_ev, h->stream));
  }
  // Ticks may run from here on: the copy to the caller and the commit wait for the passes only, on the checkpoint stream.
  AM_CUDA(h, cudaEventSynchronize(h->ck_ev));
  const uint64_t m = n ? h->ckd_acc_h[1] : 0;
  const CkptLayout L = ckpt_layout(m, hd.switches, ckd_start(m));
  std::vector<CkptZone> zones;
  int rc = ckpt_marked_zones(h, (const uint32_t*)(h->ck_meta_h + 1), "am_sweep_checkpoint_delta", &zones);
  if (rc != AM_OK) return rc;
  hd.n_changed = m;
  rc = ckpt_seal(h, (char*)buf, cap, &hd, L, m, true, zones, len_out);
  if (rc != AM_OK) return rc;  // (AM_E_NOSPACE: nothing committed, the next delta carries these slots again)
  // the blob is the caller's: the base image advances to it
  if (m) {
    AM_CUDA(h, launch(h, delta_commit_kernel, (unsigned)((m + 255) / 256), 256, h->ck_stream,
                      ckd_base_blob(h, n, hd.switches), ckpt_blob(h, L, m), (const uint32_t*)h->ckd_off));
    AM_CUDA(h, cudaStreamSynchronize(h->ck_stream));
  }
  h->chain_checksum = hd.checksum;
  h->chain_seq = hd.seq;
  h->chain_prev_tick = hd.prev_tick;
  *n_changed = m;
  return AM_OK;
}

int am_checkpoint_delta_info(const void* buf, uint64_t len, am_checkpoint_delta_info_t* info) {
  if (!info) return AM_E_INVAL;
  CkptHeader hd;
  CkptLayout L;
  std::vector<CkptZone> zones;
  const int rc = ckpt_parse(buf, len, true, &hd, &L, &zones);
  if (rc != AM_OK) return rc;
  *info = am_checkpoint_delta_info_t{};
  info->first_global = hd.first_global;
  info->n = hd.n;
  info->swept_end = hd.swept_end;
  info->prev_tick = hd.prev_tick;
  info->seed = hd.seed;
  info->n_changed = hd.n_changed;
  info->seq = hd.seq;
  info->parent_prev_tick = hd.parent_prev_tick;
  info->parent_checksum = hd.parent_checksum;
  info->checksum = hd.checksum;
  info->switches = hd.switches;
  info->n_zones = hd.n_zones;
  info->version = hd.version;
  info->bytes = hd.bytes;
  return AM_OK;
}

int am_sweep_restore_delta(am_sweep_t* h, const void* buf, uint64_t len) {
  if (!h || !buf) return AM_E_INVAL;
  std::lock_guard<std::mutex> ck(h->ck_mu);
  CkptRestore r;
  int rc = ckpt_restore_check(h, buf, len, true, &r);
  if (rc != AM_OK) return rc;
  const CkptHeader& hd = r.hd;
  TickGuard g(h);
  if (!g.ok) return AM_E_BUSY;
  CkptLink* link = nullptr;
  for (CkptLink& e : h->links)
    if (e.first_global == hd.first_global && e.n == hd.n) link = &e;
  if (!link || link->checksum != hd.parent_checksum) {
    h->last_error = "am_sweep_restore_delta: the delta's parent is not the last link this handle applied for its range";
    return AM_E_INVAL;
  }
  if (link->ticks != h->ticks) {
    h->last_error = "am_sweep_restore_delta: the handle ticked since it applied the delta's parent";
    return AM_E_INVAL;
  }
  rc = ckpt_restore_switches(h, hd.switches, "am_sweep_restore_delta");
  if (rc != AM_OK) return rc;
  const int64_t P = h->has_prev ? h->prev_T : INT64_MIN;
  if (P != hd.parent_prev_tick && P != hd.prev_tick) {
    h->last_error = "am_sweep_restore_delta: the handle's previous tick is neither the delta's nor its parent's";
    return AM_E_INVAL;
  }
  rc = ckpt_restore_apply(h, r);
  if (rc != AM_OK) return rc;
  link->checksum = hd.checksum;
  link->ticks = h->ticks;
  return AM_OK;
}

}  // extern "C"
