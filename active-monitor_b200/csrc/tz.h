// tz.h — named time zones for cron schedules ("CRON_TZ=Europe/Paris 0 9 * * *").
//
// robfig/cron v3.0.1 (parser.go, call site hcc.go:253) resolves the prefix with
// time.LoadLocation and evaluates the schedule in that zone.  Round 1 rejected such specs
// (AM_E_UNSUPPORTED, kind HOST_FALLBACK) and nothing evaluated them.  Now: a process-wide
// registry maps zone names to small ids (carried in bits 24..31 of a record's flags); the device
// holds one UTC offset per registered zone, refreshed only when a tick leaves the window in which
// no zone changes its offset (twice a year per zone); for a zone-bound record the kernel breaks
// T + offset down into the same one-hot TickWords it ANDs against the cron masks — still five ANDs.
//
// Zone rules come from the system's TZif files (RFC 8536; $ZONEINFO, /usr/share/zoneinfo, ... —
// the directories Go's time.LoadLocation searches): the 64-bit transition table plus the POSIX TZ
// footer for instants past the last transition (slim files carry little else).  No libc, no
// global TZ state: the oracle uses libc / zoneinfo instead, so the two share nothing.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "civil.h"
#include "tz_eval.h"

namespace amsweep_tz {

constexpr int kMaxZones = 255;  // ids 1..255; 0 = UTC / time.Local of the shipped image

// Register (or find) a zone by name.  0 ok (*id_out set; "", "UTC", "Local" -> 0); -1 the zone
// cannot be loaded (robfig: "provided bad location"); -2 registry full.
int lookup(const char* name, size_t len, int32_t* id_out);
// UTC offset (seconds east) of zone `id` at a UTC instant.  false: unknown id.
bool offset_at(int32_t id, int64_t utc, int32_t* utoff);
int count();
// The name zone `id` was registered under.  false: unknown id (0 included).
bool name_of(int32_t id, std::string* name);
// Flattened copy of the registry for the device (entry 0 = UTC) and its version (bumped on every
// registration); descs == nullptr: the version only.
uint64_t snapshot(std::vector<ZoneDesc>* descs, std::vector<int64_t>* trans, std::vector<int32_t>* off);
// The UTC offset of every registered zone at `utc` (entry 0 = UTC = 0), the instant up to which all of
// them stay what they are (the earliest next transition / daylight-rule instant of any zone: the
// sweep re-reads the registry only when a tick leaves [utc, *valid_until) or the version changes), and
// whether every offset is a whole number of minutes (the kernel may then skip the cron masks off the
// minute: the local second-of-minute equals the UTC one).  Returns the registry version.
uint64_t offsets_at(int64_t utc, std::vector<int32_t>* offs, int64_t* valid_until, bool* minute_aligned);
// A catch-up tick's window (lo, hi] of UTC seconds as calendar boxes (civil.h, window_boxes), per zone:
// the window is split where the zone changes its offset, each constant-offset piece mapped to the zone's
// local seconds.  boxes[z * kWindowBoxes ..] for zone z = 0 (UTC) .. count(), unused entries with sec0 = 0.
// *n_zones = count() + 1.  *steady: no zone may change its offset inside the window (next_change finds no instant
// in it; a spurious one only costs the fast path) and every offset is a whole number of minutes — every zone's
// local minute starts are then the UTC ones.  false: some zone needs more than kWindowBoxes boxes.
bool window_boxes(int64_t lo, int64_t hi, std::vector<amsweep::TickWords>* boxes, uint32_t* n_zones, bool* steady);

}  // namespace amsweep_tz
