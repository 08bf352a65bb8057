// C++ test of HealthCheckReconciler::StatusWrites (include/amsweep_reconciler.hpp): one check through Succeeded, a
// Failed that runs its remedy, the remedy's Failed and the reset on the next pass, compared with the fields
// hcc.go:636-661, :663-721 and :836-851 assign.  Needs a CUDA device (run by tests/test_status_writes_cpp.py).
#include <cstdio>
#include <string>

#include "amsweep_reconciler.hpp"

using namespace amsweep;

static int failures = 0;
#define CHECK(cond)                                                          \
  do {                                                                       \
    if (!(cond)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); ++failures; } \
  } while (0)

static const int64_t T0 = 1789982100;  // 2026-09-21 09:15:00 UTC

static StatusWrite only(const std::vector<StatusWrite>& w) {
  CHECK(w.size() == 1);
  return w.empty() ? StatusWrite{} : w[0];
}

int main() {
  std::string err;
  auto r = HealthCheckReconciler::New(0, 16, &err);
  if (!r) { std::printf("no device: %s\n", err.c_str()); return 1; }
  CHECK(am_sweep_set_hold_in_flight(r->Handle(), 1) == AM_OK);
  CHECK(am_sweep_set_hold_remedy(r->Handle(), 1) == AM_OK);
  CHECK(r->EnableStatusWrites() == AM_OK);
  HealthCheck hc;
  hc.Namespace = "default";
  hc.Name = "hc";
  hc.Spec.RepeatAfterSec = 60;
  hc.Spec.Remedy.GenerateName = "remedy-";
  hc.Spec.Remedy.HasResource = true;
  hc.Status.FinishedAt = T0 - 100;
  CHECK(!r->ProcessHealthCheck(&hc, T0).has_value());
  auto due = r->Tick(T0);  // submitted: the run starts at T0
  CHECK(due.size() == 1 && (due[0].Action & AM_ACT_SUBMIT_HC));
  CHECK(r->StatusWrites(T0).empty());

  r->PostResult(hc.Key(), Succeeded);  // hcc.go:636-648
  r->Tick(T0 + 5);
  StatusWrite w = only(r->StatusWrites(T0 + 5));
  CHECK(w.Key == "default/hc" && w.Status.Status == "Succeeded");
  CHECK(w.Status.StartedAt == T0 && w.Status.FinishedAt == T0 + 5 && !w.Status.LastFailedAt);
  CHECK(w.Status.SuccessCount == 1 && w.Status.TotalHealthCheckRuns == 1 && w.Status.RemedyStatus.empty());

  r->Tick(T0 + 65);  // submitted again
  r->PostResult(hc.Key(), Failed);  // hcc.go:663-675, the remedy runs (:712-719)
  r->Tick(T0 + 70);
  w = only(r->StatusWrites(T0 + 70));
  CHECK(w.Status.Status == "Failed" && w.Status.StartedAt == T0 + 65 && w.Status.FinishedAt == T0 + 70);
  CHECK(w.Status.LastFailedAt == T0 + 70 && w.Status.FailedCount == 1 && (w.Detail.action & AM_ACT_RUN_REMEDY));

  r->PostResult(hc.Key(), None, Failed);  // the remedy's Failed, hcc.go:836-848
  r->Tick(T0 + 80);
  w = only(r->StatusWrites(T0 + 80));
  CHECK(w.Status.RemedyStatus == "Failed" && w.Status.RemedyStartedAt == T0 + 70);
  CHECK(w.Status.RemedyFinishedAt == T0 + 80 && w.Status.RemedyLastFailedAt == T0 + 80);
  CHECK(w.Status.RemedyFailedCount == 1 && w.Status.RemedyTotalRuns == 1 && w.Status.Status.empty());

  r->Tick(T0 + 140);  // submitted again (finishedAt T0 + 70)
  r->PostResult(hc.Key(), Succeeded);  // the pass resets the remedy, hcc.go:649-660
  r->Tick(T0 + 150);
  w = only(r->StatusWrites(T0 + 150));
  CHECK(w.Status.Status == "Succeeded" && w.Status.StartedAt == T0 + 140);
  CHECK(w.Status.RemedyStatus == "HealthCheck Passed so Remedy is reset" && w.Status.RemedyTotalRuns == 0);
  CHECK(!w.Status.RemedyStartedAt && !w.Status.RemedyLastFailedAt);
  if (failures) { std::printf("%d failures\n", failures); return 1; }
  std::printf("ok\n");
  return 0;
}
