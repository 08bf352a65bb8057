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

// am_sweep_checkpoint: element j = slot first + j, one thread each (a warp's 32 slots make one word of the bit section).
__global__ void __launch_bounds__(256) checkpoint_pack_kernel(const CkptState s, const CkptBlob b, uint64_t first,
                                                             unsigned long long* sum, uint32_t* zones) {
  __shared__ uint32_t s_zones[8];
  if (threadIdx.x < 8) s_zones[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const bool in = j < b.n;
  const uint64_t i = first + j;
  uint64_t acc = 0;
  if (in) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (ck_elem(k) == 8) {
        const uint64_t v = reinterpret_cast<const uint64_t*>(s.col[k])[i];
        reinterpret_cast<uint64_t*>(b.p + b.off[k])[j] = v;
        acc += ck_term(b, k, j, v);
      } else {
        const uint32_t v = reinterpret_cast<const uint32_t*>(s.col[k])[i];
        reinterpret_cast<uint32_t*>(b.p + b.off[k])[j] = v;
        acc += ck_term(b, k, j, v);
        if (k == 6) mark_zone(s_zones, v);
      }
    }
    if (b.off[kCkSecWfTimeout]) {
      const int32_t w = s.wf_timeout[i];
      const int64_t d = s.deadline[i];
      reinterpret_cast<int32_t*>(b.p + b.off[kCkSecWfTimeout])[j] = w;
      reinterpret_cast<int64_t*>(b.p + b.off[kCkSecDeadline])[j] = d;
      acc += ck_term(b, kCkSecWfTimeout, j, w) + ck_term(b, kCkSecDeadline, j, d);
    }
    if (b.off[kCkSecSince]) {
      const int64_t v = s.since[i];
      reinterpret_cast<int64_t*>(b.p + b.off[kCkSecSince])[j] = v;
      acc += ck_term(b, kCkSecSince, j, v);
    }
    if (b.off[kCkSecDetApplied]) {
      const uint8_t a = s.det_applied[i];
      const int64_t t = s.det_start[i];
      reinterpret_cast<uint8_t*>(b.p + b.off[kCkSecDetApplied])[j] = a;
      reinterpret_cast<int64_t*>(b.p + b.off[kCkSecDetStart])[j] = t;
      acc += ckpt_mix((b.off[kCkSecDetApplied] + j) * 8, a) + ck_term(b, kCkSecDetStart, j, t);
    }
    if (b.off[kCkSecWait]) {
      const int64_t v = s.wait[i];
      reinterpret_cast<int64_t*>(b.p + b.off[kCkSecWait])[j] = v;
      acc += ck_term(b, kCkSecWait, j, v);
    }
  }
  if (b.off[kCkSecChanged]) {  // (warp-uniform)
    const uint32_t bit = in ? (s.changed[i >> 5] >> (i & 31)) & 1u : 0u;
    const uint32_t word = __ballot_sync(kFull, bit);
    if ((threadIdx.x & 31) == 0 && j < b.n) reinterpret_cast<uint32_t*>(b.p + b.off[kCkSecChanged])[j >> 5] = word;
    if (in) acc += ckpt_mix(b.off[kCkSecChanged] * 8 + j, bit);
  }
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
        case 1: acc += ckpt_mix((b.off[k] + j) * 8, ck_blob_get<uint8_t>(b, k, j)); break;
        default: acc += ckpt_mix(b.off[k] * 8 + j, (ck_blob_get<uint32_t>(b, k, j >> 5) >> (j & 31)) & 1u);
      }
    }
  }
  ck_reduce(acc, s_zones, sum, zones);
}

// The zone ids of the restoring process, by the blob's id (the blob's table resolved with am_tz_lookup).
struct ZoneLut {
  uint8_t id[256];
};

// am_sweep_restore: element j to slot first + j, every section the handle has; zone ids rewritten through `lut`.  A
// handle with the timeout state restoring a blob without it gets no timeout and no deadline for the slots.
__global__ void __launch_bounds__(256) checkpoint_scatter_kernel(const CkptState s, const CkptBlob b, uint64_t first,
                                                                const ZoneLut lut) {
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j >= b.n) return;
  const uint64_t i = first + j;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (ck_elem(k) == 8) {
      reinterpret_cast<uint64_t*>(s.col[k])[i] = ck_blob_get<uint64_t>(b, k, j);
    } else {
      uint32_t v = ck_blob_get<uint32_t>(b, k, j);
      if (k == 6 && zone_bound(v)) v = (v & ~AM_F_TZ_MASK) | ((uint32_t)lut.id[v >> AM_F_TZ_SHIFT] << AM_F_TZ_SHIFT);
      reinterpret_cast<uint32_t*>(s.col[k])[i] = v;
    }
  }
  if (s.wf_timeout) {
    const bool has = b.off[kCkSecWfTimeout] != 0;
    const int64_t d = has ? ck_blob_get<int64_t>(b, kCkSecDeadline, j) : kNoDeadline;
    s.wf_timeout[i] = has ? ck_blob_get<int32_t>(b, kCkSecWfTimeout, j) : 0;
    s.deadline[i] = d;
    if (d != kNoDeadline) atomicMin(&s.seg_deadline[i / kRecPerWarp], biased_key(d));
  }
  if (s.since) s.since[i] = ck_blob_get<int64_t>(b, kCkSecSince, j);
  if (s.changed) {
    const uint32_t m = 1u << (i & 31);
    if ((ck_blob_get<uint32_t>(b, kCkSecChanged, j >> 5) >> (j & 31)) & 1u) atomicOr(&s.changed[i >> 5], m);
    else atomicAnd(&s.changed[i >> 5], ~m);
  }
  if (s.det_applied) {
    s.det_applied[i] = ck_blob_get<uint8_t>(b, kCkSecDetApplied, j);
    s.det_start[i] = ck_blob_get<int64_t>(b, kCkSecDetStart, j);
  }
  if (s.wait) s.wait[i] = ck_blob_get<int64_t>(b, kCkSecWait, j);
}

}  // namespace amsweep
