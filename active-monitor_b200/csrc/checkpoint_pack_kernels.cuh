// checkpoint_pack_kernels.cuh — packed checkpoints (DESIGN.md section 6 item 23, "Packed format").  A packed blob
// (format version 2) holds the sections of the version-1 blob it decodes to, cut into blocks of kCkpBlock elements,
// each block in the smallest of five encodings, with a directory of one entry per block.  The encode runs over the
// staging area a pack pass filled (and a delta's offsets), the decode writes the staging area back at the version-1
// layout, and the version-1 checksum is verified on what the decode wrote: these kernels add nothing to the checksum.
// Element values are the elements' bits sign-extended to 64 bits ("the element's signed type"); every order below is
// that signed order.
#pragma once
#ifndef AMSWEEP_EMULATE  // tests/emu compiles this file for the CPU (cuda_emu.h supplies the model)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "admission_kernels.cuh"  // (adm_block_scan)
#include "checkpoint_kernels.cuh"

namespace amsweep {

constexpr uint32_t kCkpBlock = 1024;               // elements per block (the last block of a section may hold fewer)
constexpr int kCkpThreads = 256;                   // threads per block's CTA
constexpr int kCkpMaxSecs = kCkSections + 1;       // a delta's offset section, then the sections
constexpr uint32_t kCkpDictMax = 256;              // distinct values a DICT block may hold
enum CkpMode : uint32_t { kCkpRaw, kCkpConst, kCkpFor, kCkpSparse, kCkpDict, kCkpModes };  // (the tie order)

// A directory entry: the payload's byte offset from the payload's start, the mode, the bit width, and the dictionary's
// size (DICT) or the present elements (SPARSE), 0 otherwise.
struct CkpEntry {
  uint64_t off;
  uint8_t mode, width;
  uint16_t aux;
  uint32_t zero;
};
static_assert(sizeof(CkpEntry) == 16, "directory entry: 16 bytes");

// The sections a packed blob encodes, in blob order: element 0 of each (device), its elements, their bytes, the
// section's "none" value (SPARSE), and the first block of each (blk0[n] = the blocks in all).  The change bits are a
// section of u32 words.
struct CkpSecs {
  char* p[kCkpMaxSecs];
  uint64_t cnt[kCkpMaxSecs];
  uint64_t blk0[kCkpMaxSecs + 1];
  int64_t none[kCkpMaxSecs];
  uint32_t esize[kCkpMaxSecs];
  int n;
};

// the bits needed for x (0 for 0)
AM_HD uint32_t ckp_nbits(uint64_t x) {
  uint32_t b = 0;
  for (int s = 32; s; s >>= 1)
    if (x >> s) {
      x >>= s;
      b += s;
    }
  return b + (x != 0);
}
// the code width of a dictionary of k values
AM_HD uint32_t ckp_code_bits(uint32_t k) { return k <= 1 ? 0u : ckp_nbits(k - 1); }
// bytes of the u64 words that hold `bits` bits
AM_HD uint64_t ckp_words(uint64_t bits) { return (bits + 63) / 64 * 8; }

// The payload bytes of a block of cnt elements of esize bytes in `mode` with width w and aux:
//   RAW    the elements verbatim, padded to 8 B
//   CONST  the value (8 B)
//   FOR    the minimum (8 B), then cnt w-bit offsets from it
//   SPARSE a presence bitmap (bit i of word i / 64: element i is not the section's none value), the least present
//          element (8 B; 0 when none is present), then aux w-bit offsets from it, one per present element in order
//   DICT   aux values ascending, esize bytes each, padded to 8 B, then cnt w-bit codes (w = ckp_code_bits(aux))
// w-bit fields are packed from bit 0 of u64 word 0 on, field r at bits [r w, r w + w), across word edges.
AM_HD uint64_t ckp_bytes(uint32_t mode, uint32_t w, uint32_t aux, uint64_t cnt, uint32_t esize) {
  switch (mode) {
    case kCkpRaw: return (cnt * esize + 7) / 8 * 8;
    case kCkpConst: return 8;
    case kCkpFor: return 8 + ckp_words(cnt * w);
    case kCkpSparse: return ckp_words(cnt) + 8 + ckp_words((uint64_t)aux * w);
    default: return ((uint64_t)aux * esize + 7) / 8 * 8 + ckp_words(cnt * w);
  }
}

// Whether an entry's mode, width and aux fit a block of cnt elements of esize bytes (the decoder reads only those).
AM_HD bool ckp_entry_ok(const CkpEntry& e, uint64_t cnt, uint32_t esize) {
  const uint32_t full = 8 * esize;
  switch (e.mode) {
    case kCkpRaw: return e.width == full && e.aux == 0 && e.zero == 0;
    case kCkpConst: return e.width == 0 && e.aux == 0 && e.zero == 0;
    case kCkpFor: return e.width <= full && e.aux == 0 && e.zero == 0;
    case kCkpSparse: return e.width <= full && e.aux <= cnt && e.zero == 0;
    case kCkpDict:
      return e.aux >= 1 && e.aux <= kCkpDictMax && e.aux <= cnt && e.width == ckp_code_bits(e.aux) && e.zero == 0;
    default: return false;
  }
}

// the section of block b, its first element and its elements
__device__ __forceinline__ int ckp_sec_of(const CkpSecs& S, uint64_t b, uint64_t* j0, uint32_t* cnt) {
  int s = 0;
  while (b >= S.blk0[s + 1]) ++s;
  *j0 = (b - S.blk0[s]) * kCkpBlock;
  const uint64_t left = S.cnt[s] - *j0;
  *cnt = left < kCkpBlock ? (uint32_t)left : kCkpBlock;
  return s;
}

__device__ __forceinline__ int64_t ckp_load(const char* p, uint32_t esize, uint64_t j) {
  return esize == 8 ? reinterpret_cast<const int64_t*>(p)[j]
         : esize == 4 ? (int64_t)reinterpret_cast<const int32_t*>(p)[j]
                      : (int64_t)reinterpret_cast<const int8_t*>(p)[j];
}
__device__ __forceinline__ void ckp_store(char* p, uint32_t esize, uint64_t j, int64_t v) {
  if (esize == 8) reinterpret_cast<int64_t*>(p)[j] = v;
  else if (esize == 4) reinterpret_cast<uint32_t*>(p)[j] = (uint32_t)v;
  else reinterpret_cast<uint8_t*>(p)[j] = (uint8_t)v;
}
AM_HD uint64_t ckp_mask(uint32_t w) { return w >= 64 ? ~0ull : (1ull << w) - 1; }

// Field r of width w of the packed words `in`.
__device__ __forceinline__ uint64_t ckp_field(const uint64_t* in, uint64_t r, uint32_t w) {
  if (!w) return 0;
  const uint64_t pos = r * w;
  const uint32_t sh = (uint32_t)(pos & 63);
  uint64_t v = in[pos >> 6] >> sh;
  if (sh + w > 64) v |= in[(pos >> 6) + 1] << (64 - sh);
  return v & ckp_mask(w);
}

// Block-wide: fields 0..count-1 of width w (code(r)) as packed u64 words at `out`; each thread assembles whole words.
template <class F>
__device__ __forceinline__ void ckp_put_fields(uint64_t* out, uint32_t count, uint32_t w, F code) {
  if (!w) return;
  const uint32_t nw = (uint32_t)(((uint64_t)count * w + 63) / 64);
  for (uint32_t z = threadIdx.x; z < nw; z += blockDim.x) {
    const int64_t lo = (int64_t)z * 64;
    uint64_t word = 0;
    for (uint32_t r = (uint32_t)(lo / w); r < count && (int64_t)r * w < lo + 64; ++r) {
      const uint64_t c = code(r) & ckp_mask(w);
      const int64_t sh = (int64_t)r * w - lo;  // (-w, 64)
      word |= sh >= 0 ? c << sh : c >> -sh;
    }
    out[z] = word;
  }
}
// Block-wide: count elements of esize bytes (v[i]'s low bytes) verbatim as u64 words, zero-padded.
__device__ __forceinline__ void ckp_put_elems(uint64_t* out, const int64_t* v, uint32_t count, uint32_t esize) {
  const uint32_t per = 8 / esize, nw = (count + per - 1) / per;
  for (uint32_t z = threadIdx.x; z < nw; z += blockDim.x) {
    uint64_t word = 0;
    for (uint32_t r = 0; r < per; ++r) {
      const uint32_t i = z * per + r;
      if (i < count) word |= ((uint64_t)v[i] & ckp_mask(8 * esize)) << (8 * esize * r);
    }
    out[z] = word;
  }
}

// Block-wide bitonic sort of s[0..kCkpBlock) ascending (the caller fills past the block's elements with INT64_MAX, so
// its first cnt entries are its elements in order).
__device__ __forceinline__ void ckp_sort(int64_t* s) {
  __syncthreads();
  for (uint32_t k = 2; k <= kCkpBlock; k <<= 1)
    for (uint32_t j = k >> 1; j; j >>= 1) {
      for (uint32_t t = threadIdx.x; t < kCkpBlock / 2; t += blockDim.x) {
        const uint32_t i = (t / j) * 2 * j + t % j;
        const int64_t a = s[i], b = s[i + j];
        if ((a > b) == ((i & k) == 0)) {
          s[i] = b;
          s[i + j] = a;
        }
      }
      __syncthreads();
    }
}

// Block-wide: the distinct values of the sorted s[0..cnt) to dict[0..k), ascending; returns k.  Thread t owns
// elements 4t..4t+3.
__device__ __forceinline__ uint32_t ckp_distinct(const int64_t* s, uint32_t cnt, int64_t* dict, uint32_t* s_warp) {
  constexpr uint32_t per = kCkpBlock / kCkpThreads;
  const uint32_t i0 = threadIdx.x * per;
  uint32_t mine = 0;
  for (uint32_t i = i0; i < i0 + per; ++i) mine += i < cnt && (i == 0 || s[i] != s[i - 1]);
  uint32_t k;
  uint32_t at = adm_block_scan(mine, s_warp, &k);
  if (k <= kCkpDictMax)
    for (uint32_t i = i0; i < i0 + per; ++i)
      if (i < cnt && (i == 0 || s[i] != s[i - 1])) dict[at++] = s[i];
  __syncthreads();
  return k;
}

// Pass 1, one CTA per block: the block's elements, their bounds, the present ones' and (when it can win) the distinct
// values; the smallest mode, first in kCkpRaw.. order on a tie, to dir[b] (offset 0 until pass 3), its size in words
// to words[b] (scan_groups_kernel's input) and its base value (CONST's value, FOR's or SPARSE's minimum) to base[b].
__global__ void __launch_bounds__(kCkpThreads) ckp_size_kernel(const CkpSecs S, CkpEntry* dir, uint32_t* words,
                                                               int64_t* base) {
  __shared__ int64_t s_v[kCkpBlock];
  __shared__ int64_t s_dict[kCkpDictMax];
  __shared__ int64_t s_r[4][kCkpThreads / 32];
  __shared__ uint32_t s_warp[kCkpThreads / 32];
  const uint64_t b = blockIdx.x;
  uint64_t j0;
  uint32_t cnt;
  const int s = ckp_sec_of(S, b, &j0, &cnt);
  const uint32_t es = S.esize[s];
  const int64_t none = S.none[s];
  int64_t mn = INT64_MAX, mx = INT64_MIN, pmn = INT64_MAX, pmx = INT64_MIN;
  uint32_t present = 0;
  for (uint32_t i = threadIdx.x; i < kCkpBlock; i += blockDim.x) {
    int64_t v = INT64_MAX;
    if (i < cnt) {
      v = ckp_load(S.p[s], es, j0 + i);
      mn = v < mn ? v : mn;
      mx = v > mx ? v : mx;
      if (v != none) {
        ++present;
        pmn = v < pmn ? v : pmn;
        pmx = v > pmx ? v : pmx;
      }
    }
    s_v[i] = v;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const int64_t a = (int64_t)__shfl_xor_sync(kFull, (unsigned long long)mn, d);
    const int64_t c = (int64_t)__shfl_xor_sync(kFull, (unsigned long long)mx, d);
    const int64_t e = (int64_t)__shfl_xor_sync(kFull, (unsigned long long)pmn, d);
    const int64_t f = (int64_t)__shfl_xor_sync(kFull, (unsigned long long)pmx, d);
    mn = a < mn ? a : mn;
    mx = c > mx ? c : mx;
    pmn = e < pmn ? e : pmn;
    pmx = f > pmx ? f : pmx;
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    s_r[0][warp] = mn;
    s_r[1][warp] = mx;
    s_r[2][warp] = pmn;
    s_r[3][warp] = pmx;
  }
  (void)adm_block_scan(present, s_warp, &present);  // (also the barrier that publishes s_r)
  for (int k = 0; k < kCkpThreads / 32; ++k) {
    mn = s_r[0][k] < mn ? s_r[0][k] : mn;
    mx = s_r[1][k] > mx ? s_r[1][k] : mx;
    pmn = s_r[2][k] < pmn ? s_r[2][k] : pmn;
    pmx = s_r[3][k] > pmx ? s_r[3][k] : pmx;
  }
  if (!present) pmn = pmx = 0;
  uint64_t best = ckp_bytes(kCkpRaw, 0, 0, cnt, es);
  uint32_t mode = kCkpRaw, w = 8 * es, aux = 0;
  int64_t bv = 0;
  auto consider = [&](uint32_t m, uint32_t wm, uint32_t am, int64_t vm) {
    const uint64_t bytes = ckp_bytes(m, wm, am, cnt, es);
    if (bytes < best) {
      best = bytes;
      mode = m;
      w = wm;
      aux = am;
      bv = vm;
    }
  };
  if (mn == mx) consider(kCkpConst, 0, 0, mn);
  consider(kCkpFor, ckp_nbits((uint64_t)mx - (uint64_t)mn), 0, mn);
  consider(kCkpSparse, ckp_nbits((uint64_t)pmx - (uint64_t)pmn), present, pmn);
  // DICT with k >= 2 takes at least one word of dictionary and one bit per element (k == 1 is CONST, which wins the
  // tie): sort only when that can beat the best so far (block-uniform)
  if (best > 8 + ckp_words(cnt)) {
    ckp_sort(s_v);
    const uint32_t k = ckp_distinct(s_v, cnt, s_dict, s_warp);
    if (k <= kCkpDictMax) consider(kCkpDict, ckp_code_bits(k), k, 0);
  }
  if (threadIdx.x == 0) {
    dir[b] = CkpEntry{0, (uint8_t)mode, (uint8_t)w, (uint16_t)aux, 0};
    words[b] = (uint32_t)(best / 8);
    base[b] = bv;
  }
}

// Pass 3 (after scan_groups_kernel turned the sizes into word offsets), one CTA per block: the block's payload at
// payload + 8 prefix[b] in the mode pass 1 chose, and the entry's offset.
__global__ void __launch_bounds__(kCkpThreads) ckp_write_kernel(const CkpSecs S, CkpEntry* dir,
                                                                const uint32_t* __restrict__ prefix,
                                                                const int64_t* __restrict__ base, char* payload) {
  __shared__ int64_t s_v[kCkpBlock];
  __shared__ int64_t s_d[kCkpBlock];
  __shared__ int64_t s_dict[kCkpDictMax];
  __shared__ uint16_t s_idx[kCkpBlock];
  __shared__ uint32_t s_warp[kCkpThreads / 32];
  const uint64_t b = blockIdx.x;
  uint64_t j0;
  uint32_t cnt;
  const int s = ckp_sec_of(S, b, &j0, &cnt);
  const uint32_t es = S.esize[s];
  const int64_t none = S.none[s];
  const CkpEntry e = dir[b];
  const uint32_t w = e.width;
  const int64_t bv = base[b];
  uint64_t* out = reinterpret_cast<uint64_t*>(payload + (uint64_t)prefix[b] * 8);
  for (uint32_t i = threadIdx.x; i < kCkpBlock; i += blockDim.x) s_v[i] = i < cnt ? ckp_load(S.p[s], es, j0 + i) : INT64_MAX;
  __syncthreads();
  if (threadIdx.x == 0) dir[b].off = (uint64_t)prefix[b] * 8;
  switch (e.mode) {
    case kCkpRaw: ckp_put_elems(out, s_v, cnt, es); break;
    case kCkpConst:
      if (threadIdx.x == 0) out[0] = (uint64_t)bv;
      break;
    case kCkpFor:
      if (threadIdx.x == 0) out[0] = (uint64_t)bv;
      ckp_put_fields(out + 1, cnt, w, [&](uint32_t r) { return (uint64_t)s_v[r] - (uint64_t)bv; });
      break;
    case kCkpSparse: {
      const uint32_t nbm = (cnt + 63) / 64;
      for (uint32_t q = threadIdx.x; q < nbm; q += blockDim.x) {
        uint64_t word = 0;
        for (uint32_t r = 0; r < 64 && q * 64 + r < cnt; ++r) word |= (uint64_t)(s_v[q * 64 + r] != none) << r;
        out[q] = word;
      }
      // the present elements' ranks: thread t owns elements 4t..4t+3
      constexpr uint32_t per = kCkpBlock / kCkpThreads;
      const uint32_t i0 = threadIdx.x * per;
      uint32_t mine = 0, total;
      for (uint32_t i = i0; i < i0 + per; ++i) mine += i < cnt && s_v[i] != none;
      uint32_t at = adm_block_scan(mine, s_warp, &total);
      for (uint32_t i = i0; i < i0 + per; ++i)
        if (i < cnt && s_v[i] != none) s_idx[at++] = (uint16_t)i;
      __syncthreads();
      if (threadIdx.x == 0) out[nbm] = (uint64_t)bv;
      ckp_put_fields(out + nbm + 1, e.aux, w, [&](uint32_t r) { return (uint64_t)s_v[s_idx[r]] - (uint64_t)bv; });
      break;
    }
    default: {  // DICT
      for (uint32_t i = threadIdx.x; i < kCkpBlock; i += blockDim.x) s_d[i] = s_v[i];
      ckp_sort(s_d);
      const uint32_t k = ckp_distinct(s_d, cnt, s_dict, s_warp);  // (== e.aux)
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        uint32_t lo = 0, hi = k;  // the value's index in the dictionary
        while (hi - lo > 1) {
          const uint32_t mid = (lo + hi) / 2;
          if (s_dict[mid] <= s_v[i]) lo = mid;
          else hi = mid;
        }
        s_idx[i] = (uint16_t)lo;
      }
      __syncthreads();
      ckp_put_elems(out, s_dict, k, es);
      ckp_put_fields(out + ((uint64_t)k * es + 7) / 8, cnt, w, [&](uint32_t r) { return (uint64_t)s_idx[r]; });
    }
  }
}

// A restore's first pass over a packed blob's directory (n_blocks entries, payload_bytes of payload), one thread per
// entry: the mode, width and aux fit the block (ckp_entry_ok), the first payload starts at 0 and each ends where the
// next starts, the last at payload_bytes.  *bad |= 1 otherwise.
__global__ void __launch_bounds__(256) ckp_validate_kernel(const CkpSecs S, const CkpEntry* __restrict__ dir,
                                                           uint64_t payload_bytes, uint32_t* bad) {
  const uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t nb = S.blk0[S.n];
  if (b >= nb) return;
  uint64_t j0;
  uint32_t cnt;
  const int s = ckp_sec_of(S, b, &j0, &cnt);
  const CkpEntry e = dir[b];
  bool ok = ckp_entry_ok(e, cnt, S.esize[s]) && e.off <= payload_bytes && (b || e.off == 0);
  if (ok) ok = e.off + ckp_bytes(e.mode, e.width, e.aux, cnt, S.esize[s]) == (b + 1 < nb ? dir[b + 1].off : payload_bytes);
  if (!ok) atomicOr(bad, 1u);
}

// ... then one CTA per block, unless the validation refused the directory: the block's elements to their version-1
// places.  A SPARSE bitmap whose bits do not count aux present elements, or a DICT code past the dictionary, raises
// *bad (2) and is not followed.
__global__ void __launch_bounds__(kCkpThreads) ckp_decode_kernel(const CkpSecs S, const CkpEntry* __restrict__ dir,
                                                                 const char* __restrict__ payload, uint32_t* bad) {
  __shared__ uint32_t s_pre[kCkpBlock / 64 + 1];
  if (*bad & 1u) return;  // (grid-uniform: the validation's flag, complete before this pass)
  const uint64_t b = blockIdx.x;
  uint64_t j0;
  uint32_t cnt;
  const int s = ckp_sec_of(S, b, &j0, &cnt);
  const uint32_t es = S.esize[s];
  const CkpEntry e = dir[b];
  const uint32_t w = e.width;
  const uint64_t* in = reinterpret_cast<const uint64_t*>(payload + e.off);
  char* dst = S.p[s];
  switch (e.mode) {
    case kCkpRaw:
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x)
        ckp_store(dst, es, j0 + i, ckp_load(reinterpret_cast<const char*>(in), es, i));
      break;
    case kCkpConst:
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) ckp_store(dst, es, j0 + i, (int64_t)in[0]);
      break;
    case kCkpFor:
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x)
        ckp_store(dst, es, j0 + i, (int64_t)(in[0] + ckp_field(in + 1, i, w)));
      break;
    case kCkpSparse: {
      const uint32_t nbm = (cnt + 63) / 64;
      if (threadIdx.x == 0) {
        uint32_t at = 0;
        for (uint32_t q = 0; q < nbm; ++q) {
          s_pre[q] = at;
          const uint64_t m = q + 1 < nbm || cnt % 64 == 0 ? ~0ull : (1ull << (cnt % 64)) - 1;
          const uint64_t word = in[q] & m;
          at += (uint32_t)(__popc((uint32_t)word) + __popc((uint32_t)(word >> 32)));
        }
        s_pre[kCkpBlock / 64] = at;
      }
      __syncthreads();
      if (s_pre[kCkpBlock / 64] != e.aux) {  // (block-uniform)
        if (threadIdx.x == 0) atomicOr(bad, 2u);
        return;
      }
      const int64_t none = S.none[s];
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        const uint64_t word = in[i / 64], below = word & ((1ull << (i % 64)) - 1);
        int64_t v = none;
        if ((word >> (i % 64)) & 1u) {
          const uint32_t r = s_pre[i / 64] + (uint32_t)(__popc((uint32_t)below) + __popc((uint32_t)(below >> 32)));
          v = (int64_t)(in[nbm] + ckp_field(in + nbm + 1, r, w));
        }
        ckp_store(dst, es, j0 + i, v);
      }
      break;
    }
    default: {  // DICT
      const uint64_t* codes = in + ((uint64_t)e.aux * es + 7) / 8;
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        const uint64_t c = ckp_field(codes, i, w);
        if (c >= e.aux) {
          atomicOr(bad, 2u);
          continue;
        }
        ckp_store(dst, es, j0 + i, ckp_load(reinterpret_cast<const char*>(in), es, c));
      }
    }
  }
}

}  // namespace amsweep
