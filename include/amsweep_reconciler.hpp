// amsweep_reconciler.hpp — header-only C++17 mirror of the reference controller's surface
// for the schedule-evaluation path, on top of the C-ABI (amsweep.h).
//
// The reference is Go (internal/controllers/healthcheck_controller.go, "hcc.go"); no Go
// toolchain exists in the build image, so this is the host side "in the reference's shape"
// in C++: the same names, argument meaning and error behaviour as
//
//     NewHealthCheckReconciler           hcc.go:152
//     (*HealthCheckReconciler).Reconcile hcc.go:170   (CR present -> process; gone -> stop timer :175-186)
//     ProcessSpec                        the spec path of a Reconcile for a check already placed: the
//                                                     library keeps its status (am_sweep_update_spec)
//     processHealthCheck                 hcc.go:225   (ladder :227/:238/:251/:264, error on bad cron :254-257,
//                                                      Spec.RepeatAfterSec set from the cron schedule :262)
//     GetTimerByName                     hcc.go:1480  (the armed re-run timer of a check)
//     watchWorkflowReschedule results    hcc.go:635/:662, watchRemedyWorkflow :821/:836 -> PostResult
//
// It is a facade for tests and for readers of INTEGRATION.md, not a second implementation:
// every decision is taken by libamsweep (am_healthcheck_classify on the host, the sweep
// kernels on the device).  Keys are namespace/name (SURVEY B.4 N4: the reference keys its
// timer map by bare name; the collision is deliberately not reproduced).
#pragma once

#include <cstdint>
#include <memory>
#include <optional>
#include <string>
#include <unordered_map>
#include <vector>

#include "amsweep.h"

namespace amsweep {

// The fields of api/v1alpha1.HealthCheck that the path reads or writes
// (healthcheck_types.go:32-66); everything else stays in the Go object.
struct RemedyWorkflow {
  std::string GenerateName;
  bool HasResource = false;   // Resource != nil
  int64_t Timeout = 0;        // workflowtimeout
  bool HasRBACRules = false;  // RBACRules != nil
  bool IsEmpty() const {      // healthcheck_types.go:104-106
    return am_remedy_is_empty(GenerateName.size(), !HasResource, Timeout, !HasRBACRules) != 0;
  }
};

struct HealthCheckSpec {
  int64_t RepeatAfterSec = 0;
  struct { std::string Cron; } Schedule;
  struct { bool HasResource = true; } Workflow;  // Workflow.Resource != nil
  RemedyWorkflow Remedy;                         // RemedyWorkflow
  int64_t RemedyRunsLimit = 0, RemedyResetInterval = 0;
};

struct HealthCheckStatus {
  std::optional<int64_t> FinishedAt, RemedyFinishedAt;  // *metav1.Time as unix seconds
  int64_t SuccessCount = 0, FailedCount = 0, TotalHealthCheckRuns = 0;
  int64_t RemedySuccessCount = 0, RemedyFailedCount = 0, RemedyTotalRuns = 0;
  std::string Status;  // GetStatus: "Stopped" | ""; StatusWrites: also "Succeeded" | "Failed"
  // written by StatusWrites only (nullopt / "": not assigned by the tick, or set to nil by a remedy reset)
  std::optional<int64_t> StartedAt, LastFailedAt, RemedyStartedAt, RemedyLastFailedAt;
  std::string RemedyStatus;
};

// One status write of a tick (StatusWrites): the check and the fields hcc.go assigns for what the tick applied.
struct StatusWrite {
  std::string Key;
  HealthCheckStatus Status;
  am_change_detail_t Detail;
};

struct HealthCheck {
  std::string Namespace, Name;
  HealthCheckSpec Spec;
  HealthCheckStatus Status;
  std::string Key() const { return Namespace + "/" + Name; }
};

struct Due {
  std::string Key;
  uint32_t Action;  // AM_ACT_* bits
};

enum Phase : uint8_t { None = AM_PHASE_NONE, Succeeded = AM_PHASE_SUCCEEDED, Failed = AM_PHASE_FAILED };

class HealthCheckReconciler {
 public:
  // NewHealthCheckReconciler (hcc.go:152).  `err` receives the reason on failure (no GPU:
  // there is no CPU fallback).
  static std::unique_ptr<HealthCheckReconciler> New(int device, uint64_t capacity, std::string* err = nullptr) {
    am_sweep_t* h = nullptr;
    int rc = am_sweep_create(&h, device, capacity, 0);
    if (rc != AM_OK) {
      if (err) *err = std::string(am_strerror(rc)) + ": " + am_last_error_detail(nullptr);
      return nullptr;
    }
    return std::unique_ptr<HealthCheckReconciler>(new HealthCheckReconciler(h, capacity));
  }
  ~HealthCheckReconciler() { am_sweep_destroy(h_); }
  HealthCheckReconciler(const HealthCheckReconciler&) = delete;
  HealthCheckReconciler& operator=(const HealthCheckReconciler&) = delete;

  // processHealthCheck (hcc.go:225).  Returns the error the reference returns (bad cron,
  // :254-257); on a cron schedule sets hc->Spec.RepeatAfterSec as :262 does.  A paused check
  // (:238) and a check without Workflow.Resource (:227) are not errors.
  std::optional<std::string> ProcessHealthCheck(HealthCheck* hc, int64_t now) {
    am_record_t rec;
    // r.GetTimerByName(name) != nil (hcc.go:264): a timer exists once a result of this check was
    // applied (hcc.go:745-752) and survives re-Reconciles of the same process; a fresh reconciler
    // (restart, hcc.go:161) has none
    bool armed = false;
    am_record_t cur;
    if (slots_.count(hc->Key()) && ReadRecord(hc->Key(), &cur)) armed = (cur.flags & AM_F_TIMER_ARMED) != 0;
    if (auto err = Record(hc, armed, now, &rec)) return err;
    const uint64_t slot = SlotFor(hc->Key());
    am_sweep_upsert(h_, 1, &slot, &rec);
    return std::nullopt;
  }

  // The spec path of a Reconcile (am_sweep_update_spec) for a check already placed: only hc->Spec is taken, the
  // library keeps the check's status.  A Reconcile that a status write enqueued, or a restart's re-list with the
  // status etcd holds, then rolls back no result the library applied or has staged since.  Reads nothing from the
  // device.  A check not placed yet goes through ProcessHealthCheck.  Errors and RepeatAfterSec as there.
  std::optional<std::string> ProcessSpec(HealthCheck* hc, int64_t now) {
    auto it = slots_.find(hc->Key());
    if (it == slots_.end()) return ProcessHealthCheck(hc, now);
    am_record_t rec;
    if (auto err = Record(hc, false, now, &rec)) return err;
    am_sweep_update_spec(h_, 1, &it->second, &rec);
    return std::nullopt;
  }

  // Reconcile (hcc.go:170): hc == nullptr means the CR was not found (:175-186): stop its timer.
  std::optional<std::string> Reconcile(const std::string& key, HealthCheck* hc, int64_t now) {
    if (hc == nullptr) {
      auto it = slots_.find(key);
      if (it != slots_.end()) {
        am_sweep_remove(h_, 1, &it->second);
        free_.push_back(it->second);
        names_[it->second].clear();
        slots_.erase(it);
      }
      return std::nullopt;
    }
    return ProcessHealthCheck(hc, now);
  }

  // Terminal workflow phase seen by the watch loops (hcc.go:635/:662; remedy :821/:836).
  void PostResult(const std::string& key, Phase phase, Phase remedy = None) {
    auto it = slots_.find(key);
    if (it == slots_.end()) return;
    uint8_t p = phase, r = remedy;
    am_sweep_post_result(h_, 1, &it->second, &p, &r);
  }

  // One tick of the sweep: every decision for every check at `now`.
  std::vector<Due> Tick(int64_t now, am_tick_stats_t* stats = nullptr) {
    idx_.resize(capacity_);
    act_.resize(capacity_);
    uint64_t n = 0;
    am_tick_stats_t st{};
    last_rc_ = am_sweep_tick(h_, now, 0, idx_.data(), act_.data(), capacity_, &n, &st);
    if (stats) *stats = st;
    std::vector<Due> out;
    if (last_rc_ != AM_OK) return out;
    out.reserve(n);
    for (uint64_t k = 0; k < n; ++k) out.push_back(Due{names_[idx_[k]], act_[k]});
    return out;
  }

  // GetTimerByName (hcc.go:1480): the time at which the check's re-run timer fires
  // (finishedAt + repeatAfterSec, hcc.go:751), or nullopt when there is none (unknown check,
  // paused, cron schedule without a fixed interval).
  std::optional<int64_t> GetTimerByName(const std::string& key) {
    am_record_t r;
    if (!ReadRecord(key, &r)) return std::nullopt;
    const uint32_t kind = r.flags & AM_KIND_MASK;
    if ((r.flags & AM_F_TOMBSTONE) || !(r.flags & AM_F_TIMER_ARMED) || (kind != AM_KIND_INTERVAL && kind != AM_KIND_CRON_EVERY))
      return std::nullopt;
    return r.finished_at + r.ras;
  }

  // Status as updateHealthCheckStatus (hcc.go:1445) would persist it.
  std::optional<HealthCheckStatus> GetStatus(const std::string& key) {
    am_record_t r;
    if (!ReadRecord(key, &r) || (r.flags & AM_F_TOMBSTONE)) return std::nullopt;
    HealthCheckStatus s;
    if (r.finished_at) s.FinishedAt = r.finished_at;
    if (r.remedy_finished_at) s.RemedyFinishedAt = r.remedy_finished_at;
    s.SuccessCount = r.success;
    s.FailedCount = r.failed;
    s.TotalHealthCheckRuns = (int64_t)r.success + r.failed;  // hcc.go:643/:671
    s.RemedySuccessCount = r.remedy_success;
    s.RemedyFailedCount = r.remedy_failed;
    s.RemedyTotalRuns = r.remedy_total;
    if ((r.flags & AM_KIND_MASK) == AM_KIND_STOPPED && (r.flags & AM_F_STOPPED_REPORTED)) s.Status = "Stopped";
    return s;
  }

  // Status changes with their details (am_sweep_set_track_changes + am_sweep_set_change_details), for StatusWrites.
  int EnableStatusWrites() {
    const int rc = am_sweep_set_track_changes(h_, 1);
    return rc != AM_OK ? rc : am_sweep_set_change_details(h_, 1);
  }

  // After a tick at `now` (EnableStatusWrites first): the status writes updateHealthCheckStatus (hcc.go:1445) would
  // persist, one per check the tick changed, built from am_sweep_last_changes and am_sweep_last_change_details alone.
  // The counters and TotalHealthCheckRuns are the check's columns.  As the watch loops assign them:
  //   Succeeded (hcc.go:636-661): Status, StartedAt = then, FinishedAt = now; on the reset (AM_ACT_RESET_ON_PASS) the
  //     remedy timestamps are nil and RemedyStatus = "HealthCheck Passed so Remedy is reset";
  //   Failed (:663-721, a timeout's too, :627-632): Status, StartedAt = then, FinishedAt = LastFailedAt = now; on the
  //     interval reset (AM_ACT_RESET_ON_INTERVAL) RemedyStatus = "RemedyResetInterval elapsed so Remedy is reset";
  //   a remedy phase (:821-851), when the tick applied it (alone, or behind a Failed that runs the remedy):
  //     RemedyStatus, RemedyStartedAt = then, RemedyFinishedAt = now, and RemedyLastFailedAt = now for a Failed;
  //   AM_CHG_STOPPED: Status = "Stopped".
  // `then` is the detail's start; a field it leaves at INT64_MIN (the hold off, or no run seen) is not written.
  std::vector<StatusWrite> StatusWrites(int64_t now) {
    std::vector<StatusWrite> out;
    uint64_t n = 0;
    int rc = am_sweep_last_changes(h_, 0, nullptr, nullptr, 0, &n);
    if ((rc != AM_OK && rc != AM_E_NOSPACE) || n == 0) return out;
    std::vector<uint64_t> idx(n), idx2(n);
    std::vector<am_change_detail_t> det(n);
    std::vector<uint32_t> flags(n);
    std::vector<int64_t> fa(n), rfa(n);
    std::vector<int32_t> sc(n), fc(n), rs(n), rf(n), rt(n);
    am_record_cols_t c{};
    c.flags = flags.data(); c.finished_at = fa.data(); c.remedy_finished_at = rfa.data();
    c.success = sc.data(); c.failed = fc.data(); c.remedy_success = rs.data(); c.remedy_failed = rf.data();
    c.remedy_total = rt.data();
    if (am_sweep_last_changes(h_, 0, idx.data(), &c, n, &n) != AM_OK) return out;
    if (am_sweep_last_change_details(h_, 0, idx2.data(), det.data(), n, &n) != AM_OK) return out;
    const int64_t kNone = INT64_MIN;
    for (uint64_t k = 0; k < n; ++k) {
      const am_change_detail_t& d = det[k];
      StatusWrite w{names_[idx[k]], {}, d};
      HealthCheckStatus& s = w.Status;
      s.SuccessCount = sc[k]; s.FailedCount = fc[k]; s.TotalHealthCheckRuns = (int64_t)sc[k] + fc[k];
      s.RemedySuccessCount = rs[k]; s.RemedyFailedCount = rf[k]; s.RemedyTotalRuns = rt[k];
      const bool ok = (d.applied & AM_CHG_SUCCEEDED) != 0, fail = !ok && (d.applied & AM_CHG_FAILED) != 0;
      if (ok || fail) {
        s.Status = ok ? "Succeeded" : "Failed";
        if (d.started != kNone) s.StartedAt = d.started;
        s.FinishedAt = now;
        if (fail) s.LastFailedAt = now;
      }
      if (ok && (d.action & AM_ACT_RESET_ON_PASS)) s.RemedyStatus = "HealthCheck Passed so Remedy is reset";
      if (fail && (d.action & AM_ACT_RESET_ON_INTERVAL)) s.RemedyStatus = "RemedyResetInterval elapsed so Remedy is reset";
      const bool rem = (d.applied & (AM_CHG_REMEDY_SUCCEEDED | AM_CHG_REMEDY_FAILED)) != 0 &&
                       (!(ok || fail) || (fail && (d.action & AM_ACT_RUN_REMEDY)));
      if (rem) {
        const bool rok = (d.applied & AM_CHG_REMEDY_SUCCEEDED) != 0;
        s.RemedyStatus = rok ? "Succeeded" : "Failed";
        if (d.remedy_started != kNone) s.RemedyStartedAt = d.remedy_started;
        s.RemedyFinishedAt = now;
        if (!rok) s.RemedyLastFailedAt = now;
      }
      if (d.applied & AM_CHG_STOPPED) s.Status = "Stopped";
      out.push_back(std::move(w));
    }
    return out;
  }

  int LastTickError() const { return last_rc_; }
  am_sweep_t* Handle() { return h_; }

 private:
  HealthCheckReconciler(am_sweep_t* h, uint64_t cap) : h_(h), capacity_(cap) { names_.resize(cap); }

  // processHealthCheck's ladder on the host: the record of *hc, or the error the reference returns.
  static std::optional<std::string> Record(HealthCheck* hc, bool armed, int64_t now, am_record_t* rec) {
    std::string perr;
    int rc = Classify(*hc, armed, rec, &perr);
    if (rc == AM_E_UNSUPPORTED) return std::string("unsupported on the device path: ") + perr;
    if (rc != AM_OK) return std::string(am_strerror(rc));
    const uint32_t kind = rec->flags & AM_KIND_MASK;
    if (kind == AM_KIND_PARSE_ERROR) return perr.empty() ? std::string("fail to parse cron") : perr;
    if (kind == AM_KIND_CRON_SPEC || kind == AM_KIND_CRON_EVERY) {
      am_cron_t c;
      am_cron_parse(hc->Spec.Schedule.Cron.data(), hc->Spec.Schedule.Cron.size(), &c, nullptr, 0);
      hc->Spec.RepeatAfterSec = am_cron_repeat_after_sec(&c, now);  // hcc.go:262
    }
    return std::nullopt;
  }

  static int Classify(const HealthCheck& hc, bool timer_armed, am_record_t* rec, std::string* perr) {
    am_healthcheck_t in{};
    in.timer_armed = timer_armed ? 1u : 0u;
    in.repeat_after_sec = hc.Spec.RepeatAfterSec;
    in.cron = hc.Spec.Schedule.Cron.data();
    in.cron_len = hc.Spec.Schedule.Cron.size();
    in.has_resource = hc.Spec.Workflow.HasResource;
    in.has_remedy = !hc.Spec.Remedy.IsEmpty();
    in.remedy_runs_limit = hc.Spec.RemedyRunsLimit;
    in.remedy_reset_interval = hc.Spec.RemedyResetInterval;
    if (hc.Status.FinishedAt) { in.finished_at = *hc.Status.FinishedAt; in.finished_at_set = 1; }
    if (hc.Status.RemedyFinishedAt) { in.remedy_finished_at = *hc.Status.RemedyFinishedAt; in.remedy_finished_at_set = 1; }
    in.success_count = hc.Status.SuccessCount;
    in.failed_count = hc.Status.FailedCount;
    in.remedy_success_count = hc.Status.RemedySuccessCount;
    in.remedy_failed_count = hc.Status.RemedyFailedCount;
    in.remedy_total_runs = hc.Status.RemedyTotalRuns;
    int rc = am_healthcheck_classify(&in, rec);
    if ((rec->flags & AM_KIND_MASK) == AM_KIND_PARSE_ERROR || rc == AM_E_UNSUPPORTED) {
      am_cron_t c;
      char buf[256] = {0};
      am_cron_parse(in.cron, in.cron_len, &c, buf, sizeof buf);
      *perr = buf;
    }
    return rc;
  }

  uint64_t SlotFor(const std::string& key) {
    auto it = slots_.find(key);
    if (it != slots_.end()) return it->second;
    uint64_t s;
    if (!free_.empty()) { s = free_.back(); free_.pop_back(); }
    else s = next_++;
    slots_[key] = s;
    names_[s] = key;
    return s;
  }

  bool ReadRecord(const std::string& key, am_record_t* r) {
    auto it = slots_.find(key);
    if (it == slots_.end()) return false;
    am_record_cols_t c{};
    c.minute = &r->minute; c.hour = &r->hour; c.dom = &r->dom; c.month = &r->month; c.dow = &r->dow;
    c.ras = &r->ras; c.flags = &r->flags; c.finished_at = &r->finished_at;
    c.runs_limit = &r->runs_limit; c.reset_interval = &r->reset_interval;
    c.success = &r->success; c.failed = &r->failed; c.remedy_success = &r->remedy_success;
    c.remedy_failed = &r->remedy_failed; c.remedy_total = &r->remedy_total;
    c.remedy_finished_at = &r->remedy_finished_at;
    // staged events are applied by the next tick: read what the device holds
    return am_sweep_read(h_, 0, 1, &it->second, &c) == AM_OK;
  }

  am_sweep_t* h_;
  uint64_t capacity_;
  uint64_t next_ = 0;
  int last_rc_ = AM_OK;
  std::unordered_map<std::string, uint64_t> slots_;
  std::vector<std::string> names_;
  std::vector<uint64_t> free_;
  std::vector<uint64_t> idx_;
  std::vector<uint32_t> act_;
};

}  // namespace amsweep
