// civil.h — UTC broken-down time from a unix second, shared by host code and
// the sweep kernel (closed-form days→civil conversion; no libc, no tables).
//
// The reference reaches the same quantities through Go's time package inside
// robfig/cron's SpecSchedule.Next (call site hcc.go:262): t.Second(),
// t.Minute(), t.Hour(), t.Day(), t.Month(), t.Weekday() with Sunday = 0.
#pragma once
#include <stdint.h>

#ifndef INT64_MIN
#define INT64_MIN (-9223372036854775807ll - 1)
#endif

#if defined(__CUDACC__)
#define AM_HD __host__ __device__ __forceinline__
#else
#define AM_HD inline
#endif

namespace amsweep {

struct CivilTime {
  int32_t sec, min, hour, dom, month, dow;  // dom 1-31, month 1-12, dow 0=Sunday
  int64_t year;
};

// floor-div split of a unix second into (days since epoch, second of day)
AM_HD void split_days(int64_t t, int64_t& days, int32_t& sod) {
  int64_t d = t / 86400;
  int64_t s = t - d * 86400;
  if (s < 0) { s += 86400; d -= 1; }
  days = d;
  sod = (int32_t)s;
}

// proleptic Gregorian (what Go's time package uses), era-based closed form
AM_HD void civil_from_days(int64_t days, int64_t& y, int32_t& m, int32_t& d) {
  int64_t z = days + 719468;  // shift epoch to 0000-03-01
  int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  uint32_t doe = (uint32_t)(z - era * 146097);                                 // [0, 146096]
  uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;        // [0, 399]
  uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);                      // [0, 365]
  uint32_t mp = (5 * doy + 2) / 153;                                           // [0, 11]
  d = (int32_t)(doy - (153 * mp + 2) / 5 + 1);
  m = (int32_t)(mp < 10 ? mp + 3 : mp - 9);
  y = (int64_t)yoe + era * 400 + (m <= 2);
}

AM_HD int64_t days_from_civil(int64_t y, int32_t m, int32_t d) {
  y -= m <= 2;
  int64_t era = (y >= 0 ? y : y - 399) / 400;
  uint32_t yoe = (uint32_t)(y - era * 400);
  uint32_t doy = (153u * (uint32_t)(m > 2 ? m - 3 : m + 9) + 2u) / 5u + (uint32_t)d - 1u;
  uint32_t doe = yoe * 365u + yoe / 4u - yoe / 100u + doy;
  return era * 146097 + (int64_t)doe - 719468;
}

AM_HD int32_t weekday_from_days(int64_t days) {  // 1970-01-01 was a Thursday (4)
  return (int32_t)(((days % 7) + 11) % 7);
}

AM_HD CivilTime civil_from_unix(int64_t t) {
  CivilTime c;
  int64_t days;
  int32_t sod;
  split_days(t, days, sod);
  c.hour = sod / 3600;
  c.min = (sod % 3600) / 60;
  c.sec = sod % 60;
  civil_from_days(days, c.year, c.month, c.dom);
  c.dow = weekday_from_days(days);
  return c;
}

// The tick's broken-down time as one-hot words: what a 64-bit cron field mask
// is ANDed with.  sec0 is the Second field test (ParseStandard pins Second to
// 1<<0, SURVEY A.1), so a 5-field schedule can only fire when sec0 != 0.
struct TickWords {
  uint64_t minute, hour, dom, month, dow;
  uint32_t sec0;
  uint32_t pad;
};

AM_HD TickWords tick_words_from_unix(int64_t t) {
  CivilTime c = civil_from_unix(t);
  TickWords w;
  w.minute = 1ull << c.min;
  w.hour = 1ull << c.hour;
  w.dom = 1ull << c.dom;
  w.month = 1ull << c.month;
  w.dow = 1ull << c.dow;
  w.sec0 = (c.sec == 0) ? 1u : 0u;
  w.pad = 0;
  return w;
}

// A catch-up tick (AM_SWEEP_CATCH_UP) asks whether a schedule fires at SOME second of a window.  The
// minute starts of a window form a few calendar boxes: one day, a range of hours, a range of minutes (a
// partial first hour, whole hours, a partial last hour).  A box is a TickWords whose hour and minute words
// are range masks instead of one-hot ones, with sec0 = 1: inside a box the hour and the minute tests are
// independent, so cron_matches against it is exactly "fires at some minute start of the box".
constexpr int kWindowBoxes = 16;  // boxes per zone of one catch-up tick

AM_HD int64_t floor_div(int64_t a, int64_t b) {
  const int64_t q = a / b;
  return q - ((a % b != 0) && ((a < 0) != (b < 0)));
}
AM_HD uint64_t bit_range(int32_t lo, int32_t hi) { return (2ull << hi) - (1ull << lo); }  // bits lo..hi, hi < 63

// Append the boxes of the minute starts in the LOCAL seconds (lo, hi] to out[*n ..].  False (out and *n
// then unspecified) when they would not fit in `cap` boxes.  At most three boxes per day the window touches.
AM_HD bool window_boxes(int64_t lo, int64_t hi, TickWords* out, int* n, int cap) {
  const int64_t m0 = floor_div(lo, 60) + 1, m1 = floor_div(hi, 60);  // minute numbers of the first and last start
  if (m0 > m1) return true;
  for (int64_t day = floor_div(m0, 1440); day <= floor_div(m1, 1440); ++day) {
    const int32_t a = (int32_t)((m0 > day * 1440 ? m0 : day * 1440) - day * 1440);         // minute of the day
    const int32_t b = (int32_t)((m1 < day * 1440 + 1439 ? m1 : day * 1440 + 1439) - day * 1440);
    int64_t y;
    int32_t mo, d;
    civil_from_days(day, y, mo, d);
    TickWords w;
    w.dom = 1ull << d;
    w.month = 1ull << mo;
    w.dow = 1ull << weekday_from_days(day);
    w.sec0 = 1;
    w.pad = 0;
    const int32_t ha = a / 60, hb = b / 60, ma = a % 60, mb = b % 60;
    // rows: [hour, hour] x [minute lo, minute hi]; a partial first / last hour that is whole joins the middle
    int32_t rows[3][4];
    int nr = 0;
    if (ha == hb) {
      rows[nr][0] = ha; rows[nr][1] = ha; rows[nr][2] = ma; rows[nr][3] = mb; ++nr;
    } else {
      const int32_t full_lo = ma == 0 ? ha : ha + 1, full_hi = mb == 59 ? hb : hb - 1;
      if (ma != 0) { rows[nr][0] = ha; rows[nr][1] = ha; rows[nr][2] = ma; rows[nr][3] = 59; ++nr; }
      if (full_lo <= full_hi) { rows[nr][0] = full_lo; rows[nr][1] = full_hi; rows[nr][2] = 0; rows[nr][3] = 59; ++nr; }
      if (mb != 59) { rows[nr][0] = hb; rows[nr][1] = hb; rows[nr][2] = 0; rows[nr][3] = mb; ++nr; }
    }
    for (int k = 0; k < nr; ++k) {
      if (*n >= cap) return false;
      w.hour = bit_range(rows[k][0], rows[k][1]);
      w.minute = bit_range(rows[k][2], rows[k][3]);
      out[(*n)++] = w;
    }
  }
  return true;
}

#if defined(__CUDA_ARCH__)
#define AM_CTZ64(x) (__ffsll((long long)(x)) - 1)
#else
#define AM_CTZ64(x) __builtin_ctzll(x)
#endif

constexpr int64_t kNoNextFire = INT64_MIN;  // robfig's zero time: nothing within five years

// SpecSchedule.Next(t) of robfig/cron v3.0.1 (call site hcc.go:262) for a whole
// UTC second t: the first activation strictly after t, or kNoNextFire when the
// year would pass year(t+1s)+5.  Not the Go field-increment loop: a forward scan
// over days with bit tricks (jump over months whose bit is clear; first set
// hour/minute bit by count-trailing-zeros), shared by the host helper
// am_cron_next and the device kernel next_fire_kernel.
AM_HD int64_t cron_next_utc(uint64_t minute, uint64_t hour, uint64_t dom, uint64_t month,
                            uint64_t dow, int64_t t) {
  const uint64_t mins = minute & ((1ull << 60) - 1);
  const uint64_t hrs = hour & ((1ull << 24) - 1);
  if (!mins || !hrs) return kNoNextFire;
  const bool star = ((dom | dow) >> 63) != 0;
  const int64_t start = t + 1;
  int64_t day0;
  int32_t sod;
  split_days(start, day0, sod);
  int64_t y;
  int32_t m, d;
  civil_from_days(day0, y, m, d);
  const int64_t year_limit = y + 5;
  const int32_t mod0 = (sod + 59) / 60;  // first candidate minute-of-day on the starting day
  for (int64_t day = day0;; ++day) {
    civil_from_days(day, y, m, d);
    if (y > year_limit) return kNoNextFire;
    if (!((month >> m) & 1)) {  // jump to the 1st of the next month
      int64_t ny = y;
      int32_t nm = m + 1;
      if (nm == 13) { nm = 1; ++ny; }
      day = days_from_civil(ny, nm, 1) - 1;
      continue;
    }
    const bool a = (dom >> d) & 1, b = (dow >> weekday_from_days(day)) & 1;
    if (!(star ? (a && b) : (a || b))) continue;  // robfig dayMatches
    if (day != day0)
      return day * 86400 + (int64_t)AM_CTZ64(hrs) * 3600 + (int64_t)AM_CTZ64(mins) * 60;
    if (mod0 >= 1440) continue;  // start was in the last minute of the day
    const int32_t h0 = mod0 / 60, m0 = mod0 % 60;
    if ((hrs >> h0) & 1) {
      const uint64_t later = mins >> m0;
      if (later) return day * 86400 + h0 * 3600 + (int64_t)(m0 + AM_CTZ64(later)) * 60;
    }
    const uint64_t hl = (h0 + 1 < 24) ? (hrs >> (h0 + 1)) : 0;
    if (hl) return day * 86400 + (int64_t)(h0 + 1 + AM_CTZ64(hl)) * 3600 + (int64_t)AM_CTZ64(mins) * 60;
  }
}

// hcc.go:262  RepeatAfterSec = int(Next(now).Sub(now')/time.Second) + 1 for a real
// clock (0 < ns): whole seconds from floor(now) to the next activation; when Next is
// the zero time Sub saturates: int(minDuration/Second) + 1.
AM_HD int64_t repeat_after_from_next(int64_t next, int64_t t) {
  return next == kNoNextFire ? -9223372036ll + 1 : next - t;
}

}  // namespace amsweep
