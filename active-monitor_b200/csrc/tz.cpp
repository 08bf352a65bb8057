// tz.cpp — TZif reader + POSIX TZ footer rules + the zone registry (see tz.h).
#include "tz.h"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace amsweep_tz {
namespace {

using amsweep::civil_from_days;
using amsweep::days_from_civil;
using amsweep::split_days;
using amsweep::weekday_from_days;

struct Zone {
  std::string name;
  std::vector<int64_t> trans;  // transition instants, ascending
  std::vector<int32_t> off;    // off[i] is in force from trans[i] on
  int32_t off_first = 0;       // before the first transition
  bool has_footer = false, has_dst = false;
  int32_t std_off = 0, dst_off = 0;  // seconds EAST of UTC
  Rule start{-1, 0, 0, 0, 7200}, end{-1, 0, 0, 0, 7200};
};

ZoneDesc desc_of(const Zone& z, uint32_t begin) {
  ZoneDesc d{};
  d.trans_begin = begin;
  d.trans_count = (uint32_t)z.trans.size();
  d.off_first = z.off_first;
  d.has_footer = z.has_footer;
  d.has_dst = z.has_dst;
  d.std_off = z.std_off;
  d.dst_off = z.dst_off;
  d.start = z.start;
  d.end = z.end;
  return d;
}

int64_t be64(const unsigned char* p) {
  uint64_t v = 0;
  for (int i = 0; i < 8; ++i) v = (v << 8) | p[i];
  return (int64_t)v;
}
int32_t be32(const unsigned char* p) {
  return (int32_t)(((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3]);
}

// ---- POSIX TZ string: std offset [dst [offset] [,start[/time],end[/time]]] ----
bool tz_name(const char*& s) {
  if (*s == '<') {
    ++s;
    while (*s && *s != '>') ++s;
    if (*s != '>') return false;
    ++s;
    return true;
  }
  int n = 0;
  while ((*s >= 'A' && *s <= 'Z') || (*s >= 'a' && *s <= 'z')) { ++s; ++n; }
  return n >= 3;
}
bool tz_hms(const char*& s, int32_t& out, bool allow_sign) {
  int sign = 1;
  if (allow_sign && (*s == '+' || *s == '-')) { if (*s == '-') sign = -1; ++s; }
  if (*s < '0' || *s > '9') return false;
  int32_t v[3] = {0, 0, 0};
  for (int k = 0; k < 3; ++k) {
    int n = 0;
    while (*s >= '0' && *s <= '9' && n < 4) { v[k] = v[k] * 10 + (*s - '0'); ++s; ++n; }
    if (n == 0) return false;
    if (*s != ':' || k == 2) break;
    ++s;
  }
  out = sign * (v[0] * 3600 + v[1] * 60 + v[2]);
  return true;
}
bool tz_rule(const char*& s, Rule& r) {
  if (*s == 'M') {
    ++s;
    r.kind = 2;
    int* f[3] = {&r.a, &r.b, &r.c};
    for (int k = 0; k < 3; ++k) {
      int v = 0, n = 0;
      while (*s >= '0' && *s <= '9') { v = v * 10 + (*s - '0'); ++s; ++n; }
      if (!n) return false;
      *f[k] = v;
      if (k < 2) { if (*s != '.') return false; ++s; }
    }
    if (r.a < 1 || r.a > 12 || r.b < 1 || r.b > 5 || r.c > 6) return false;
  } else {
    r.kind = 1;
    if (*s == 'J') { r.kind = 0; ++s; }
    int v = 0, n = 0;
    while (*s >= '0' && *s <= '9') { v = v * 10 + (*s - '0'); ++s; ++n; }
    if (!n) return false;
    r.a = v;
  }
  r.time = 7200;
  if (*s == '/') { ++s; if (!tz_hms(s, r.time, true)) return false; }
  return true;
}
bool parse_footer(const std::string& f, Zone& z) {
  const char* s = f.c_str();
  int32_t west = 0;
  if (!tz_name(s) || !tz_hms(s, west, true)) return false;
  z.std_off = -west;
  z.has_dst = false;
  if (*s == 0) return true;
  if (!tz_name(s)) return false;
  z.dst_off = z.std_off + 3600;
  if (*s && *s != ',') { if (!tz_hms(s, west, true)) return false; z.dst_off = -west; }
  if (*s == 0) return true;  // "std offset dst" without rules: POSIX leaves it to the implementation; treat as no DST
  if (*s != ',') return false;
  ++s;
  if (!tz_rule(s, z.start) || *s != ',') return false;
  ++s;
  if (!tz_rule(s, z.end) || *s != 0) return false;
  z.has_dst = true;
  return true;
}

bool load_file(const std::string& path, Zone& z) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  std::vector<unsigned char> buf;
  unsigned char tmp[65536];
  size_t n;
  while ((n = fread(tmp, 1, sizeof tmp, f)) > 0) {
    buf.insert(buf.end(), tmp, tmp + n);
    if (buf.size() > (8u << 20)) break;
  }
  fclose(f);
  if (buf.size() < 44 || memcmp(buf.data(), "TZif", 4) != 0) return false;
  const unsigned char* p = buf.data();
  const unsigned char* end = p + buf.size();
  const int version = p[4];
  auto counts = [&](const unsigned char* h, uint32_t c[6]) { for (int k = 0; k < 6; ++k) c[k] = (uint32_t)be32(h + 20 + 4 * k); };
  uint32_t c[6];  // isutcnt, isstdcnt, leapcnt, timecnt, typecnt, charcnt
  counts(p, c);
  size_t tsz = 4;  // width of a transition time in the block we read
  const unsigned char* d = p + 44;
  if (version >= '2') {
    const size_t v1 = (size_t)c[3] * 4 + c[3] + (size_t)c[4] * 6 + c[5] + (size_t)c[2] * 8 + c[1] + c[0];
    if (d + v1 + 44 > end || memcmp(d + v1, "TZif", 4) != 0) return false;
    p = d + v1;
    counts(p, c);
    d = p + 44;
    tsz = 8;
  }
  const size_t need = (size_t)c[3] * tsz + c[3] + (size_t)c[4] * 6 + c[5] + (size_t)c[2] * (tsz + 4) + c[1] + c[0];
  if (d + need > end || c[4] == 0) return false;
  const unsigned char* times = d;
  const unsigned char* idx = times + (size_t)c[3] * tsz;
  const unsigned char* types = idx + c[3];
  std::vector<int32_t> utoff(c[4]);
  std::vector<unsigned char> isdst(c[4]);
  for (uint32_t k = 0; k < c[4]; ++k) { utoff[k] = be32(types + 6 * k); isdst[k] = types[6 * k + 4]; }
  z.trans.resize(c[3]);
  z.off.resize(c[3]);
  for (uint32_t k = 0; k < c[3]; ++k) {
    z.trans[k] = tsz == 8 ? be64(times + 8 * k) : (int64_t)be32(times + 4 * k);
    if (idx[k] >= c[4]) return false;
    z.off[k] = utoff[idx[k]];
  }
  // before the first transition: the first standard-time type (as Go's lookupFirstZone), else type 0
  z.off_first = utoff[0];
  for (uint32_t k = 0; k < c[4]; ++k) if (!isdst[k]) { z.off_first = utoff[k]; break; }
  if (c[3] == 0) z.off_first = utoff[0];
  z.has_footer = false;
  if (tsz == 8) {
    const unsigned char* ft = d + need;
    if (ft < end && *ft == '\n') {
      const unsigned char* fe = (const unsigned char*)memchr(ft + 1, '\n', (size_t)(end - ft - 1));
      if (fe && fe > ft + 1) {
        std::string footer((const char*)ft + 1, (size_t)(fe - ft - 1));
        z.has_footer = parse_footer(footer, z);
      }
    }
  }
  return true;
}

int32_t zone_offset(const Zone& z, int64_t utc) {
  return tz_zone_offset(desc_of(z, 0), z.trans.data(), z.off.data(), utc);
}

std::mutex g_mu;
std::vector<std::unique_ptr<Zone>> g_zones;  // id - 1
uint64_t g_version = 0;                      // bumped on every registration

bool valid_name(const std::string& n) {  // Go: containsDotDot, leading '/' or '\\' are "invalid location name"
  if (n.empty() || n[0] == '/' || n[0] == '\\' || n.size() > 255) return false;
  return n.find("..") == std::string::npos;
}

}  // namespace

int lookup(const char* name, size_t len, int32_t* id_out) {
  const std::string n(name ? name : "", len);
  if (n.empty() || n == "UTC" || n == "Local") { *id_out = 0; return 0; }  // time.Local == UTC in the shipped image
  if (!valid_name(n)) return -1;
  std::lock_guard<std::mutex> lk(g_mu);
  for (size_t k = 0; k < g_zones.size(); ++k)
    if (g_zones[k]->name == n) { *id_out = (int32_t)k + 1; return 0; }
  auto z = std::make_unique<Zone>();
  z->name = n;
  std::vector<std::string> dirs;
  if (const char* e = getenv("ZONEINFO")) dirs.emplace_back(e);
  dirs.insert(dirs.end(), {"/usr/share/zoneinfo", "/usr/share/lib/zoneinfo", "/usr/lib/locale/TZ", "/etc/zoneinfo"});
  bool ok = false;
  for (const std::string& d : dirs)
    if (load_file(d + "/" + n, *z)) { ok = true; break; }
  if (!ok) return -1;
  if ((int)g_zones.size() >= kMaxZones) return -2;
  g_zones.push_back(std::move(z));
  ++g_version;
  *id_out = (int32_t)g_zones.size();
  return 0;
}

bool offset_at(int32_t id, int64_t utc, int32_t* utoff) {
  if (id == 0) { *utoff = 0; return true; }
  std::lock_guard<std::mutex> lk(g_mu);
  if (id < 0 || (size_t)id > g_zones.size()) return false;
  *utoff = zone_offset(*g_zones[(size_t)id - 1], utc);
  return true;
}

uint64_t snapshot(std::vector<ZoneDesc>* descs, std::vector<int64_t>* trans, std::vector<int32_t>* off) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (descs) {
    descs->clear(); trans->clear(); off->clear();
    descs->push_back(ZoneDesc{});  // id 0 = UTC: no transitions, offset 0
    for (const auto& z : g_zones) {
      descs->push_back(desc_of(*z, (uint32_t)trans->size()));
      trans->insert(trans->end(), z->trans.begin(), z->trans.end());
      off->insert(off->end(), z->off.begin(), z->off.end());
    }
  }
  return g_version;
}

int count() {
  std::lock_guard<std::mutex> lk(g_mu);
  return (int)g_zones.size();
}

bool name_of(int32_t id, std::string* name) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (id < 1 || (size_t)id > g_zones.size()) return false;
  *name = g_zones[(size_t)id - 1]->name;
  return true;
}

namespace {
// the next instant after `utc` at which zone_offset(z, .) may change (never later than the true one)
int64_t next_change(const Zone& z, int64_t utc) {
  const size_t n = z.trans.size();
  if (n && utc < z.trans[n - 1]) {  // inside (or before) the transition table: the first transition after utc
    size_t lo = 0, hi = n;          // first index with trans > utc
    while (lo < hi) {
      const size_t mid = (lo + hi) / 2;
      if (z.trans[mid] > utc) hi = mid; else lo = mid + 1;
    }
    return z.trans[lo];
  }
  if (!z.has_footer || !z.has_dst) return INT64_MAX;
  // the footer's rule instants, and the turn of the (standard-time) year at which tz_footer_offset
  // switches to the next year's instants: years y-1 .. y+1 around utc
  int64_t days, y;
  int32_t sod, m, d;
  split_days(utc + z.std_off, days, sod);
  civil_from_days(days, y, m, d);
  int64_t best = INT64_MAX;
  for (int64_t yy = y - 1; yy <= y + 1; ++yy) {
    const int64_t c[3] = {tz_rule_local_seconds(z.start, yy) - z.std_off, tz_rule_local_seconds(z.end, yy) - z.dst_off,
                          days_from_civil(yy, 1, 1) * 86400 - z.std_off};
    for (int64_t v : c)
      if (v > utc && v < best) best = v;
  }
  return best;
}
}  // namespace

uint64_t offsets_at(int64_t utc, std::vector<int32_t>* offs, int64_t* valid_until, bool* minute_aligned) {
  std::lock_guard<std::mutex> lk(g_mu);
  offs->assign(g_zones.size() + 1, 0);
  int64_t until = INT64_MAX;
  bool aligned = true;
  for (size_t k = 0; k < g_zones.size(); ++k) {
    const int32_t off = zone_offset(*g_zones[k], utc);
    (*offs)[k + 1] = off;
    if (off % 60) aligned = false;
    const int64_t nc = next_change(*g_zones[k], utc);
    if (nc < until) until = nc;
  }
  *valid_until = until;
  *minute_aligned = aligned;
  return g_version;
}

bool window_boxes(int64_t lo, int64_t hi, std::vector<amsweep::TickWords>* boxes, uint32_t* n_zones, bool* steady) {
  std::lock_guard<std::mutex> lk(g_mu);
  const size_t nz = g_zones.size() + 1;
  *n_zones = (uint32_t)nz;
  *steady = true;
  boxes->assign(nz * amsweep::kWindowBoxes, amsweep::TickWords{});
  for (size_t k = 0; k < nz; ++k) {
    amsweep::TickWords* out = boxes->data() + k * amsweep::kWindowBoxes;
    int n = 0;
    if (k == 0) {
      if (!amsweep::window_boxes(lo, hi, out, &n, amsweep::kWindowBoxes)) return false;
      continue;
    }
    const Zone& z = *g_zones[k - 1];
    // seconds s .. e-1 of the window share one offset: the piece (s - 1, e - 1] in UTC
    for (int64_t s = lo + 1; s <= hi;) {
      const int32_t off = zone_offset(z, s);
      const int64_t nc = next_change(z, s);
      const int64_t e = nc <= hi ? nc : hi + 1;
      if (s != lo + 1 || e != hi + 1 || off % 60 != 0) *steady = false;
      if (!amsweep::window_boxes(s - 1 + off, e - 1 + off, out, &n, amsweep::kWindowBoxes)) return false;
      s = e;
    }
  }
  return true;
}

}  // namespace amsweep_tz
