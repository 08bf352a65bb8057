// checkpoint_kernels.cuh — the device passes of am_sweep_checkpoint and am_sweep_restore (DESIGN.md section 6 item 19
// and "Checkpoint format").  A blob holds, per slot of its range, one element of each present SECTION (the sixteen
// columns, the workflow timeout and deadline, since, the change bit, the detail capture), every section an array over
// the range at an 8-B aligned byte offset.  Its checksum is the sum, mod 2^64, of ckpt_mix(key, value) over every
// element (key = the element's bit offset in the blob, value = its bits zero-extended), every header word and every
// word of the zone table; the host adds the header's and the table's terms to the sum these kernels reduce.
#pragma once
#ifndef AMSWEEP_EMULATE  // tests/emu compiles this file for the CPU (cuda_emu.h supplies the model)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "sweep_kernels.cuh"  // (build_segment_planes, for the planes of a delta's slots)
#include "sweep_types.h"

namespace amsweep {

// Sections in blob order: the sixteen columns (am_record_cols_t order), then the optional ones.
enum CkptSection : int {
  kCkSecWfTimeout = 16,  // i32, with the timeout state
  kCkSecDeadline,        // i64, with the timeout state
  kCkSecSince,           // i64, while the hold is on (remedy runs as T + 2^60)
  kCkSecChanged,         // 1 bit per slot in u32 words, while tracking is on
  kCkSecDetApplied,      // u8, while details are on
  kCkSecDetStart,        // i64, while details are on
  kCkSecWait,            // i64, with the submit budget's admission state: the second since which the slot waits
  kCkSections
};
// element bytes per section (0: the bit section)
AM_HD constexpr uint32_t ck_elem(int s) {
  return (s < 5 || s == 7 || s == 15 || s == kCkSecDeadline || s == kCkSecSince || s == kCkSecDetStart ||
          s == kCkSecWait) ? 8
         : s == kCkSecChanged ? 0 : s == kCkSecDetApplied ? 1 : 4;
}

AM_HD uint64_t ckpt_mix(uint64_t key, uint64_t v) {
  uint64_t x = (v ^ (key * 0x9E3779B97F4A7C15ull)) * 0xBF58476D1CE4E5B9ull;
  return x ^ (x >> 31);
}

// A blob's sections in HBM: off[s] = byte offset of section s in the blob (0: absent; the header is at 0).  `p` is the
// blob's byte 0 (the staging area; the header itself is never there).
struct CkptBlob {
  char* p;
  uint64_t off[kCkSections];
  uint64_t n;
};

// The handle's per-slot state a blob carries; NULL where the handle has none.
struct CkptState {
  void* col[16];
  int32_t* wf_timeout;
  int64_t* deadline;
  unsigned long long* seg_deadline;  // restore only: lowered to stay a lower bound
  int64_t* since;
  uint32_t* changed;
  uint8_t* det_applied;
  int64_t* det_start;
  int64_t* wait;  // the submit budget's waiting seconds
};

template <class T>
__device__ __forceinline__ uint64_t ck_bits(T v) {
  return sizeof(T) == 8 ? (uint64_t)v : (uint64_t)(uint32_t)v;
}

// Element j of section s of the blob, and its checksum term.
template <class T>
__device__ __forceinline__ T ck_blob_get(const CkptBlob& b, int s, uint64_t j) {
  return reinterpret_cast<const T*>(b.p + b.off[s])[j];
}
template <class T>
__device__ __forceinline__ uint64_t ck_term(const CkptBlob& b, int s, uint64_t j, T v) {
  return ckpt_mix((b.off[s] + j * sizeof(T)) * 8, ck_bits(v));
}
// Bit j of the bit section s of the blob.
__device__ __forceinline__ uint32_t ck_blob_bit(const CkptBlob& b, int s, uint64_t j) {
  return (ck_blob_get<uint32_t>(b, s, j >> 5) >> (j & 31)) & 1u;
}
// Element j of section s of the blob := v; returns its checksum term.
template <class T>
__device__ __forceinline__ uint64_t ck_put(const CkptBlob& b, int s, uint64_t j, T v) {
  reinterpret_cast<T*>(b.p + b.off[s])[j] = v;
  return ck_term(b, s, j, v);
}

// Zone ids belong to 5-field schedules only (the other kinds' bits 24..31 are carried as they are).
__device__ __forceinline__ bool zone_bound(uint32_t flags) {
  return (flags & AM_KIND_MASK) == AM_KIND_CRON_SPEC && (flags >> AM_F_TZ_SHIFT) != 0;
}
__device__ __forceinline__ void mark_zone(uint32_t* s_zones, uint32_t flags) {
  if (zone_bound(flags)) atomicOr(&s_zones[flags >> (AM_F_TZ_SHIFT + 5)], 1u << ((flags >> AM_F_TZ_SHIFT) & 31u));
}

// The end of a pass: the block's zone marks (one bit per id, in shared memory) and the warps' checksum terms to global memory.
__device__ __forceinline__ void ck_reduce(uint64_t acc, uint32_t* s_zones, unsigned long long* sum, uint32_t* zones) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(kFull, (unsigned long long)acc, d);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(sum, (unsigned long long)acc);
  __syncthreads();
  if (threadIdx.x < 8 && s_zones[threadIdx.x]) atomicOr(&zones[threadIdx.x], s_zones[threadIdx.x]);
}

// The section rules of a pack, per slot: slot i of the handle to element k of every section of the blob but the bit
// section; returns the elements' checksum terms and marks the slot's zone in s_zones.
__device__ __forceinline__ uint64_t ck_pack_slot(const CkptState& s, const CkptBlob& b, uint64_t i, uint64_t k,
                                                 uint32_t* s_zones) {
  uint64_t acc = 0;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    if (ck_elem(q) == 8) {
      acc += ck_put(b, q, k, reinterpret_cast<const uint64_t*>(s.col[q])[i]);
    } else {
      const uint32_t v = reinterpret_cast<const uint32_t*>(s.col[q])[i];
      acc += ck_put(b, q, k, v);
      if (q == 6) mark_zone(s_zones, v);
    }
  }
  if (b.off[kCkSecWfTimeout]) {  // (both loads before the stores: the compiler cannot tell that they do not alias)
    const int32_t w = s.wf_timeout[i];
    const int64_t d = s.deadline[i];
    acc += ck_put(b, kCkSecWfTimeout, k, w) + ck_put(b, kCkSecDeadline, k, d);
  }
  if (b.off[kCkSecSince]) acc += ck_put(b, kCkSecSince, k, s.since[i]);
  if (b.off[kCkSecDetApplied]) {
    const uint8_t a = s.det_applied[i];
    const int64_t t = s.det_start[i];
    acc += ck_put(b, kCkSecDetApplied, k, a) + ck_put(b, kCkSecDetStart, k, t);
  }
  if (b.off[kCkSecWait]) acc += ck_put(b, kCkSecWait, k, s.wait[i]);
  return acc;
}

// ... and of the bit section, warp-collective (every lane calls it; `in`: k is one of the blob's elements): the change
// bit of slot i to bit k, a warp's 32 elements one word; returns the bit's checksum term.
__device__ __forceinline__ uint64_t ck_pack_changed(const CkptState& s, const CkptBlob& b, bool in, uint64_t i,
                                                    uint64_t k) {
  const uint32_t bit = in ? (s.changed[i >> 5] >> (i & 31)) & 1u : 0u;
  const uint32_t word = __ballot_sync(kFull, bit);
  if ((threadIdx.x & 31) == 0 && in) reinterpret_cast<uint32_t*>(b.p + b.off[kCkSecChanged])[k >> 5] = word;
  return in ? ckpt_mix(b.off[kCkSecChanged] * 8 + k, bit) : 0;
}

// am_sweep_checkpoint: element j = slot first + j, one thread each.
__global__ void __launch_bounds__(256) checkpoint_pack_kernel(const CkptState s, const CkptBlob b, uint64_t first,
                                                             unsigned long long* sum, uint32_t* zones) {
  __shared__ uint32_t s_zones[8];
  if (threadIdx.x < 8) s_zones[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const bool in = j < b.n;
  uint64_t acc = in ? ck_pack_slot(s, b, first + j, j, s_zones) : 0;
  if (b.off[kCkSecChanged]) acc += ck_pack_changed(s, b, in, first + j, j);  // (warp-uniform)
  ck_reduce(acc, s_zones, sum, zones);
}

// am_sweep_restore, before anything changes: the checksum terms of the blob's sections and the zone ids its flags use.
__global__ void __launch_bounds__(256) checkpoint_verify_kernel(const CkptBlob b, unsigned long long* sum, uint32_t* zones) {
  __shared__ uint32_t s_zones[8];
  if (threadIdx.x < 8) s_zones[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t acc = 0;
  if (j < b.n) {
    for (int k = 0; k < kCkSections; ++k) {
      if (!b.off[k]) continue;
      switch (ck_elem(k)) {
        case 8: acc += ck_term(b, k, j, ck_blob_get<uint64_t>(b, k, j)); break;
        case 4: {
          const uint32_t v = ck_blob_get<uint32_t>(b, k, j);
          acc += ck_term(b, k, j, v);
          if (k == 6) mark_zone(s_zones, v);
          break;
        }
        case 1: acc += ck_term(b, k, j, ck_blob_get<uint8_t>(b, k, j)); break;
        default: acc += ckpt_mix(b.off[k] * 8 + j, ck_blob_bit(b, k, j));
      }
    }
  }
  ck_reduce(acc, s_zones, sum, zones);
}

// The zone ids of the restoring process, by the blob's id (the blob's table resolved with am_tz_lookup).
struct ZoneLut {
  uint8_t id[256];
};

// The section rules of a restore, per slot: element k of the blob to slot i, every section the handle has; zone ids
// rewritten through `lut`.  A handle with the timeout state restoring a blob without it gets no timeout and no
// deadline for the slot.
__device__ __forceinline__ void ck_scatter_slot(const CkptState& s, const CkptBlob& b, uint64_t i, uint64_t k,
                                                const ZoneLut& lut) {
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    if (ck_elem(q) == 8) {
      reinterpret_cast<uint64_t*>(s.col[q])[i] = ck_blob_get<uint64_t>(b, q, k);
    } else {
      uint32_t v = ck_blob_get<uint32_t>(b, q, k);
      if (q == 6 && zone_bound(v)) v = (v & ~AM_F_TZ_MASK) | ((uint32_t)lut.id[v >> AM_F_TZ_SHIFT] << AM_F_TZ_SHIFT);
      reinterpret_cast<uint32_t*>(s.col[q])[i] = v;
    }
  }
  if (s.wf_timeout) {
    const bool has = b.off[kCkSecWfTimeout] != 0;
    const int64_t d = has ? ck_blob_get<int64_t>(b, kCkSecDeadline, k) : kNoDeadline;
    s.wf_timeout[i] = has ? ck_blob_get<int32_t>(b, kCkSecWfTimeout, k) : 0;
    s.deadline[i] = d;
    if (d != kNoDeadline) atomicMin(&s.seg_deadline[i / kRecPerWarp], biased_key(d));
  }
  if (s.since) s.since[i] = ck_blob_get<int64_t>(b, kCkSecSince, k);
  if (s.changed) {
    const uint32_t m = 1u << (i & 31);
    if (ck_blob_bit(b, kCkSecChanged, k)) atomicOr(&s.changed[i >> 5], m);
    else atomicAnd(&s.changed[i >> 5], ~m);
  }
  if (s.det_applied) {
    s.det_applied[i] = ck_blob_get<uint8_t>(b, kCkSecDetApplied, k);
    s.det_start[i] = ck_blob_get<int64_t>(b, kCkSecDetStart, k);
  }
  if (s.wait) s.wait[i] = ck_blob_get<int64_t>(b, kCkSecWait, k);
}

// am_sweep_restore: element j to slot first + j.
__global__ void __launch_bounds__(256) checkpoint_scatter_kernel(const CkptState s, const CkptBlob b, uint64_t first,
                                                                const ZoneLut lut) {
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j < b.n) ck_scatter_slot(s, b, first + j, j, lut);
}

// ---- delta checkpoints (am_sweep_checkpoint_delta / am_sweep_restore_delta, DESIGN.md "Delta format") ----------------
// A delta of m changed slots of a chain's range holds, after its 128-B header, the slots' offsets (u32, relative to the
// range's first slot, strictly ascending) and then every section of the root, each an array over the m slots in blob
// order.  Its checksum is the full blob's rule over that layout (the offset section's elements included).

constexpr uint64_t kCkHeaderBytes = 128;

// The sections of a blob of n slots with `switches`, from byte `start` on, each at an 8-B aligned offset; returns the
// end of the last one.  A full blob starts them at the header's end, a delta of m slots at ckd_start(m).
AM_HD uint64_t ck_layout(uint64_t n, uint32_t switches, uint64_t start, uint64_t* off) {
  uint64_t at = start;
  for (int s = 0; s < kCkSections; ++s) {
    const bool on = s < 16 || ((s == kCkSecWfTimeout || s == kCkSecDeadline) && (switches & AM_CKPT_TIMEOUTS)) ||
                    (s == kCkSecSince && (switches & AM_CKPT_HOLD)) ||
                    (s == kCkSecChanged && (switches & AM_CKPT_TRACK)) ||
                    ((s == kCkSecDetApplied || s == kCkSecDetStart) && (switches & AM_CKPT_DETAILS)) ||
                    (s == kCkSecWait && (switches & AM_CKPT_ADMISSION));
    off[s] = on ? at : 0;
    if (on) at += ((s == kCkSecChanged ? (n + 31) / 32 * 4 : n * ck_elem(s)) + 7) / 8 * 8;
  }
  return at;
}
AM_HD uint64_t ckd_start(uint64_t m) { return kCkHeaderBytes + (m * 4 + 7) / 8 * 8; }

// The diff: slot first + j of the live state against element j of the base image `b` (the previous link, in the root's
// layout over the chain's range), one thread each.  Bit j of `bits` is set iff any element a blob carries differs; a
// warp's 32 slots make one word, and each 8192-slot group's count goes to group_count (scan_groups_kernel's input).
__global__ void __launch_bounds__(256) delta_diff_kernel(const CkptState s, const CkptBlob b, uint64_t first,
                                                        uint32_t* bits, uint32_t* group_count) {
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const bool in = j < b.n;
  const uint64_t i = first + j;
  bool d = false;
  if (in) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (ck_elem(k) == 8) d |= reinterpret_cast<const uint64_t*>(s.col[k])[i] != ck_blob_get<uint64_t>(b, k, j);
      else d |= reinterpret_cast<const uint32_t*>(s.col[k])[i] != ck_blob_get<uint32_t>(b, k, j);
    }
    if (b.off[kCkSecWfTimeout])
      d |= s.wf_timeout[i] != ck_blob_get<int32_t>(b, kCkSecWfTimeout, j) ||
           s.deadline[i] != ck_blob_get<int64_t>(b, kCkSecDeadline, j);
    if (b.off[kCkSecSince]) d |= s.since[i] != ck_blob_get<int64_t>(b, kCkSecSince, j);
    if (b.off[kCkSecChanged]) d |= ((s.changed[i >> 5] >> (i & 31)) & 1u) != ck_blob_bit(b, kCkSecChanged, j);
    if (b.off[kCkSecDetApplied])
      d |= s.det_applied[i] != ck_blob_get<uint8_t>(b, kCkSecDetApplied, j) ||
           s.det_start[i] != ck_blob_get<int64_t>(b, kCkSecDetStart, j);
    if (b.off[kCkSecWait]) d |= s.wait[i] != ck_blob_get<int64_t>(b, kCkSecWait, j);
  }
  const uint32_t word = __ballot_sync(kFull, d);
  if ((threadIdx.x & 31) == 0 && in) {
    bits[j >> 5] = word;
    if (word) atomicAdd(&group_count[j / kGroupRecords], (uint32_t)__popc(word));
  }
}

// The delta's sections: changed slot k (offs[k], as list_changes_kernel wrote it from the diff's bitmap; m = *count
// of them) to element k of every section, one thread each, at the layout of a delta of m slots (its sections land in
// `dev` from byte 128 on), with the checksum terms of the offsets and the sections and the zone marks (ck_reduce).
__global__ void __launch_bounds__(256) delta_pack_kernel(const CkptState s, char* dev, uint32_t switches,
                                                        const uint32_t* __restrict__ offs,
                                                        const unsigned long long* __restrict__ count, uint64_t first,
                                                        unsigned long long* sum, uint32_t* zones) {
  __shared__ uint32_t s_zones[8];
  __shared__ CkptBlob s_b;
  const uint64_t m = *count;
  if ((uint64_t)blockIdx.x * blockDim.x >= m) return;  // (block-uniform)
  if (threadIdx.x < 8) s_zones[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    const uint64_t start = ckd_start(m);
    ck_layout(m, switches, start, s_b.off);
    s_b.p = dev + kCkHeaderBytes - start;
    s_b.n = m;
  }
  __syncthreads();
  const CkptBlob& b = s_b;
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const bool in = k < m;
  const uint64_t j = in ? offs[k] : 0;
  const uint64_t i = first + j;
  uint64_t acc = in ? ckpt_mix((kCkHeaderBytes + k * 4) * 8, j) : 0;
  if (in) acc += ck_pack_slot(s, b, i, k, s_zones);
  if (b.off[kCkSecChanged]) acc += ck_pack_changed(s, b, in, i, k);  // (block-uniform)
  ck_reduce(acc, s_zones, sum, zones);
}

// Element k of every section of the compact delta `d` to element offs[k] of the same section of the full-layout image
// `b`: the commit of a delta into the producer's base image, after the copy to the caller.
__global__ void __launch_bounds__(256) delta_commit_kernel(const CkptBlob b, const CkptBlob d,
                                                          const uint32_t* __restrict__ offs) {
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (k >= d.n) return;
  const uint64_t j = offs[k];
  for (int q = 0; q < kCkSections; ++q) {
    if (!b.off[q]) continue;
    switch (ck_elem(q)) {
      case 8: reinterpret_cast<uint64_t*>(b.p + b.off[q])[j] = ck_blob_get<uint64_t>(d, q, k); break;
      case 4: reinterpret_cast<uint32_t*>(b.p + b.off[q])[j] = ck_blob_get<uint32_t>(d, q, k); break;
      case 1: reinterpret_cast<uint8_t*>(b.p + b.off[q])[j] = ck_blob_get<uint8_t>(d, q, k); break;
      default: {
        uint32_t* w = reinterpret_cast<uint32_t*>(b.p + b.off[q]) + (j >> 5);
        const uint32_t bit = 1u << (j & 31);
        if (ck_blob_bit(d, q, k)) atomicOr(w, bit);
        else atomicAnd(w, ~bit);
      }
    }
  }
}

// am_sweep_restore_delta, before anything changes: the checksum terms of the offset section (element k at byte
// 128 + 4k) and whether it is strictly ascending and below n (*bad != 0 otherwise).
__global__ void __launch_bounds__(256) delta_offsets_verify_kernel(const uint32_t* __restrict__ offs, uint64_t m,
                                                                  uint64_t n, unsigned long long* sum,
                                                                  uint32_t* bad) {
  __shared__ uint32_t s_zones[8];
  if (threadIdx.x < 8) s_zones[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t acc = 0;
  if (k < m) {
    const uint32_t j = offs[k];
    acc = ckpt_mix((kCkHeaderBytes + k * 4) * 8, j);
    if (j >= n || (k && offs[k - 1] >= j)) atomicOr(bad, 1u);
  }
  ck_reduce(acc, s_zones, sum, nullptr);  // (no zone marks: ck_reduce touches `zones` only for marked ids)
}

// am_sweep_restore_delta: element k of the delta to slot first + offs[k], and the slot's segment marked for
// delta_planes_kernel; the slot's due word as well while the handle keeps them (`due` NULL otherwise).
__global__ void __launch_bounds__(256) delta_scatter_kernel(const CkptState s, const CkptBlob b,
                                                           const uint32_t* __restrict__ offs, uint64_t first,
                                                           const ZoneLut lut, uint32_t* seg_dirty, uint32_t* due,
                                                           int64_t due_epoch) {
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (k >= b.n) return;
  const uint64_t i = first + offs[k];
  ck_scatter_slot(s, b, i, k, lut);
  if (due) due[i] = due_word(ck_blob_get<int32_t>(b, 5, k), ck_blob_get<int64_t>(b, 7, k), due_epoch);
  seg_dirty[i / kRecPerWarp] = 1u;
}

// After delta_scatter_kernel: one warp per changed slot; the first that claims its segment's mark rebuilds the
// segment's plane words (the claim of build_planes_dirty_kernel, through the offsets).
__global__ void delta_planes_kernel(DevCols c, MaskPlanes pl, uint32_t* seg_dirty, const uint32_t* __restrict__ offs,
                                    uint64_t first, uint32_t m) {
  const uint64_t k = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (k >= m) return;  // warp-uniform
  const int lane = (int)(threadIdx.x & 31);
  const uint32_t seg = (uint32_t)((first + offs[k]) / (uint32_t)kRecPerWarp);
  const bool won = lane == 0 && atomicAnd(&seg_dirty[seg], 0u) != 0u;  // (an exchange with 0)
  if (__ballot_sync(kFull, won)) build_segment_planes(c, pl, seg, lane);
}

}  // namespace amsweep
