// The spec path of the host-side mirror (include/amsweep_reconciler.hpp, ProcessSpec): a status echo that comes back
// after a result was posted keeps that result, where the same echo through Reconcile (a full upsert) drops it.
// Run by tests/test_reconciler_spec_cpp.py, on a CUDA device and on the emulated library.
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

static HealthCheck check(const std::string& name) {
  HealthCheck hc;
  hc.Namespace = "default";
  hc.Name = name;
  hc.Spec.RepeatAfterSec = 30;
  hc.Status.FinishedAt = T0 - 100;
  hc.Status.SuccessCount = 6;
  return hc;
}

// The check is submitted at T0 and its Succeeded posted; then the Reconcile enqueued by an older status write comes
// back with that status (S = 6, finishedAt T0 - 100) before the next tick.
static void echo(HealthCheckReconciler& r, bool spec_path, HealthCheckStatus* after, size_t* due_after) {
  HealthCheck hc = check(spec_path ? "spec" : "upsert");
  CHECK(!r.Reconcile(hc.Key(), &hc, T0));
  auto due = r.Tick(T0);
  CHECK(due.size() == 1 && due[0].Key == hc.Key() && (due[0].Action & AM_ACT_SUBMIT_HC));
  r.PostResult(hc.Key(), Succeeded);
  HealthCheck stale = check(hc.Name);
  CHECK(!(spec_path ? r.ProcessSpec(&stale, T0 + 1) : r.Reconcile(stale.Key(), &stale, T0 + 1)));
  *due_after = r.Tick(T0 + 2).size();
  *after = r.GetStatus(hc.Key()).value_or(HealthCheckStatus{});
}

int main() {
  std::string err;
  for (bool spec_path : {false, true}) {
    auto r = HealthCheckReconciler::New(0, 8, &err);
    if (!r) {
      std::printf("no device: %s\n", err.c_str());
      return 1;
    }
    HealthCheckStatus s;
    size_t due = 0;
    echo(*r, spec_path, &s, &due);
    if (spec_path) {  // the result is counted, and the check is not due before T0 + 32
      CHECK(s.SuccessCount == 7 && s.FinishedAt && *s.FinishedAt == T0 + 2 && due == 0);
    } else {  // the upsert superseded it: the count rolled back and the check is due again at once
      CHECK(s.SuccessCount == 6 && s.FinishedAt && *s.FinishedAt == T0 - 100 && due == 1);
    }
  }
  {  // a check that is not placed yet goes through ProcessHealthCheck; a bad cron is the same error on both paths
    auto r = HealthCheckReconciler::New(0, 8, &err);
    HealthCheck hc = check("new");
    CHECK(!r->ProcessSpec(&hc, T0));
    CHECK(r->Tick(T0).size() == 1);
    hc.Spec.RepeatAfterSec = 0;
    hc.Spec.Schedule.Cron = "NOT_A_VALID_CRON";
    auto e = r->ProcessSpec(&hc, T0 + 1);
    CHECK(e && e->find("expected exactly 5 fields") != std::string::npos);
    hc.Spec.Schedule.Cron = "*/5 * * * *";
    CHECK(!r->ProcessSpec(&hc, T0 + 1) && hc.Spec.RepeatAfterSec == 299);  // (09:20:00, hcc.go:262)
  }
  if (failures) return 1;
  std::printf("ok\n");
  return 0;
}
