// Thread-safety of checkpoints, delta chains and restores against every other kind of call on one handle, with the
// hold, change details and a finite submit budget on: four stagers (upsert, remove, post_result, update_spec), one
// ticker that retries AM_E_BUSY, one checkpointer (chain roots, deltas with the AM_E_NOSPACE path, full checkpoints,
// am_checkpoint_delta_info), one querier (the per-slot queries, next-due, repeat-after, the launch count, the last
// tick's changes, details and admission) and one restorer, which applies the chain to a second handle and, while the
// ticker repeats one second, restores a checkpoint of a range no stager touches into the ticking handle.  Built with
// -fsanitize=thread together with the emulated library sources.  Exit code 0 and no TSan report = pass.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/amsweep.h"

namespace {

const uint64_t kCap = 1024, kQuiet = 128;  // the stagers touch slots below kCap - kQuiet only
const int64_t kT0 = 1789982100;
std::atomic<bool> g_failed{false};

void fail(const char* what, int rc) {
  std::printf("%s rc %d\n", what, rc);
  g_failed.store(true);
}

template <class F>
int retry(F&& f) {  // a call retried while it returns AM_E_BUSY
  int rc;
  while ((rc = f()) == AM_E_BUSY) std::this_thread::sleep_for(std::chrono::microseconds(50));
  return rc;
}

am_sweep_t* make_handle() {
  am_sweep_t* h = nullptr;
  if (am_sweep_create(&h, 0, kCap, 0) != AM_OK) return nullptr;
  am_sweep_set_hold_in_flight(h, 1);
  am_sweep_set_track_changes(h, 1);
  am_sweep_set_change_details(h, 1);
  am_sweep_set_submit_budget(h, 7);
  am_sweep_set_seed(h, 5);
  return h;
}

}  // namespace

int main() {
  am_sweep_t* h = make_handle();
  if (!h) { std::printf("create failed\n"); return 1; }
  am_healthcheck_t hc;
  std::memset(&hc, 0, sizeof hc);
  hc.repeat_after_sec = 5;
  hc.has_resource = 1;
  hc.finished_at_set = 1;
  hc.finished_at = kT0 - 100;
  am_record_t rec;
  if (am_healthcheck_classify(&hc, &rec) != AM_OK) return 1;
  {  // every slot swept from the start, so that the chain's range holds records
    std::vector<uint64_t> idx(kCap);
    std::vector<am_record_t> recs(kCap, rec);
    for (uint64_t i = 0; i < kCap; ++i) idx[i] = i;
    if (am_sweep_upsert(h, kCap, idx.data(), recs.data()) != AM_OK) return 1;
  }

  std::atomic<bool> stop{false};
  std::atomic<uint64_t> staged{0}, busy{0}, links{0}, applied{0}, roots{0}, restored{0}, queries{0};
  std::atomic<bool> ck_done{false};  // the checkpointer took its last blob
  std::atomic<int64_t> hold_T{INT64_MIN};  // the second the ticker repeats while a restore is due, else INT64_MIN
  std::atomic<bool> restore_done{false};
  std::mutex mu;
  std::deque<std::vector<char>> chain;  // roots and deltas for the standby, in order (a root as the first byte 'R')

  std::vector<std::thread> ts;
  for (int t = 0; t < 4; ++t)
    ts.emplace_back([&, t] {
      uint64_t x = 88172645463325252ull + (uint64_t)t;
      for (int it = 0; it < 200 && !stop.load(); ++it) {
        std::this_thread::sleep_for(std::chrono::microseconds(150));  // a flood would only test the emulator's speed
        x ^= x << 13; x ^= x >> 7; x ^= x << 17;
        const uint64_t span = kCap - kQuiet;
        uint64_t idx[3] = {x % span, (x >> 20) % span, (x >> 40) % span};
        am_record_t recs[3] = {rec, rec, rec};
        recs[1].ras = 7;
        uint8_t ph[3] = {(uint8_t)(x % 3), (uint8_t)((x >> 8) % 3), 1}, rp[3] = {0, (uint8_t)((x >> 16) % 3), 2};
        int rc;
        switch (t) {
          case 0: rc = am_sweep_upsert(h, 3, idx, recs); break;
          case 1: rc = am_sweep_remove(h, 1, idx); break;
          case 2: rc = am_sweep_post_result(h, 3, idx, ph, (x >> 60) & 1 ? rp : nullptr); break;
          default: rc = am_sweep_update_spec(h, 2, idx, recs); break;
        }
        if (rc != AM_OK) fail("stager", rc);
        staged.fetch_add(1);
      }
    });

  ts.emplace_back([&] {  // checkpointer
    std::vector<char> buf(8u << 20);
    uint64_t len = 0, nch = 0;
    for (int it = 0; it < 24 && !stop.load(); ++it) {
      int rc;
      if (it % 12 == 0) {
        rc = retry([&] { return am_sweep_checkpoint_chain(h, 0, kCap, buf.data(), buf.size(), &len); });
        if (rc != AM_OK) { fail("chain", rc); continue; }
        am_checkpoint_info_t info;
        if ((rc = am_checkpoint_info(buf.data(), len, &info)) != AM_OK || info.n != kCap) fail("checkpoint_info", rc);
        std::lock_guard<std::mutex> lk(mu);
        chain.emplace_back(1, 'R');
        chain.back().insert(chain.back().end(), buf.data(), buf.data() + len);
      } else if (it % 4 == 3) {
        rc = retry([&] { return am_sweep_checkpoint(h, 0, kCap, buf.data(), buf.size(), &len); });
        if (rc != AM_OK) fail("checkpoint", rc);
      } else {
        if (it % 5 == 1) {  // too small: nothing committed, the next delta carries the same slots
          rc = retry([&] { return am_sweep_checkpoint_delta(h, buf.data(), 16, &len, &nch); });
          if (rc != AM_E_NOSPACE || len <= 16) fail("delta, short buffer", rc);
        }
        rc = retry([&] { return am_sweep_checkpoint_delta(h, buf.data(), buf.size(), &len, &nch); });
        if (rc != AM_OK) { fail("delta", rc); continue; }
        am_checkpoint_delta_info_t info;
        if ((rc = am_checkpoint_delta_info(buf.data(), len, &info)) != AM_OK || info.n_changed != nch)
          fail("delta_info", rc);
        links.fetch_add(1);
        std::lock_guard<std::mutex> lk(mu);
        chain.emplace_back(1, 'D');
        chain.back().insert(chain.back().end(), buf.data(), buf.data() + len);
      }
      std::this_thread::sleep_for(std::chrono::microseconds(300));
    }
    ck_done.store(true);
  });

  ts.emplace_back([&] {  // querier
    std::vector<int64_t> out(kCap);
    std::vector<uint64_t> idx(kCap);
    std::vector<am_change_detail_t> det(kCap);
    uint64_t q[3] = {3, 99, kCap - 1};
    while (!stop.load()) {
      int64_t nd = 0;
      uint64_t n = 0;
      am_admission_t adm;
      const int rcs[] = {
          am_sweep_in_flight(h, 0, 3, q, out.data()),
          am_sweep_remedy_in_flight(h, 0, 64, nullptr, out.data()),
          am_sweep_deferred(h, 0, 3, q, out.data()),
          am_sweep_next_due(h, kT0, &nd),
          am_sweep_repeat_after_sec(h, kT0, 0, 64, out.data()),
          am_sweep_last_changes(h, 0, idx.data(), nullptr, kCap, &n),
          am_sweep_last_change_details(h, 0, idx.data(), det.data(), kCap, &n),
          am_sweep_last_admission(h, &adm),
      };
      for (int rc : rcs) {
        if (rc == AM_E_BUSY) busy.fetch_add(1);
        else if (rc != AM_OK) fail("query", rc);
      }
      (void)am_sweep_launch_count(h);
      (void)am_sweep_size(h);
      queries.fetch_add(1);
      std::this_thread::sleep_for(std::chrono::milliseconds(5));  // (every emulated launch costs TSan memory)
    }
  });

  ts.emplace_back([&] {  // restorer
    std::vector<char> buf(1u << 20);
    uint64_t len = 0;
    am_sweep_t* standby = nullptr;  // a fresh one for every root: a standby that applied links has the P of the last
    for (;;) {                       // one, and the source has ticked since, so it would refuse the next root
      std::vector<char> b;
      {
        std::lock_guard<std::mutex> lk(mu);
        if (!chain.empty()) {
          b.swap(chain.front());
          chain.pop_front();
        }
      }
      if (b.empty() && stop.load()) break;  // (every queued blob applied)
      if (!b.empty()) {
        if (b[0] == 'R') {
          if (standby) am_sweep_destroy(standby);
          if (!(standby = make_handle())) fail("standby create", 0);
        }
        const int rc = !standby      ? AM_E_INVAL
                       : b[0] == 'R' ? am_sweep_restore(standby, b.data() + 1, b.size() - 1)
                                     : am_sweep_restore_delta(standby, b.data() + 1, b.size() - 1);
        if (rc != AM_OK) fail(b[0] == 'R' ? "standby restore" : "standby restore_delta", rc);
        (b[0] == 'R' ? roots : applied).fetch_add(1);
      }
      const int64_t T = hold_T.load();
      if (T != INT64_MIN && !restore_done.load()) {  // the ticker repeats T: P stays T while the blob goes back in
        int rc = retry([&] { return am_sweep_checkpoint(h, kCap - kQuiet, kQuiet, buf.data(), buf.size(), &len); });
        am_checkpoint_info_t info;
        if (rc == AM_OK) rc = am_checkpoint_info(buf.data(), len, &info);
        if (rc != AM_OK || info.prev_tick != T) fail("range checkpoint", rc);
        rc = retry([&] { return am_sweep_restore(h, buf.data(), len); });
        if (rc != AM_OK) fail("restore into the ticking handle", rc);
        restored.fetch_add(1);
        restore_done.store(true);
      }
      if (b.empty()) std::this_thread::sleep_for(std::chrono::microseconds(100));
    }
    if (standby) am_sweep_destroy(standby);
  });

  std::vector<uint64_t> di(kCap);
  std::vector<uint32_t> da(kCap);
  uint64_t total = 0, tick_busy = 0, zero_steps = 0;
  int64_t T = kT0;
  for (int k = 0; (k < 40 || !ck_done.load()) && k < 1000 && !g_failed.load(); ++k) {  // (until the last blob)
    const bool repeat = k % 10 == 9;  // a run of zero-step ticks at T while a restore goes into the handle
    if (repeat) {
      restore_done.store(false);
      hold_T.store(T);
    } else {
      ++T;
    }
    for (int z = 0;; ++z) {
      uint64_t n = 0;
      am_tick_stats_t st;
      int rc;
      while ((rc = am_sweep_tick(h, T, k % 3 == 0 ? AM_SWEEP_FULL_SCAN : 0u, di.data(), da.data(), kCap, &n, &st)) ==
             AM_E_BUSY) {
        ++tick_busy;
        std::this_thread::sleep_for(std::chrono::microseconds(50));
      }
      if (rc != AM_OK) { fail("tick", rc); break; }
      if (st.n_emitted != n || st.n_records > kCap) { fail("inconsistent stats", 0); break; }
      for (uint64_t i = 1; i < n; ++i)
        if (di[i] <= di[i - 1]) { fail("list not ascending", 0); break; }
      total += n;
      if (!repeat || restore_done.load() || g_failed.load()) break;
      ++zero_steps;
      if (z > 5000) { fail("restore never landed", 0); break; }
      std::this_thread::sleep_for(std::chrono::milliseconds(2));  // (room for the restorer to take the guard)
    }
    hold_T.store(INT64_MIN);
  }
  stop.store(true);
  for (auto& t : ts) t.join();
  if (!g_failed.load() && (roots.load() != 2 || links.load() != applied.load() || restored.load() < 3))
    fail("too little done", 0);
  am_sweep_destroy(h);
  if (g_failed.load()) return 1;
  std::printf("ok %llu staged calls, %llu entries emitted, %llu zero-step ticks, %llu delta links applied to "
              "standbys of %llu roots, %llu range restores, %llu query rounds, AM_E_BUSY: %llu ticks, %llu queries\n",
              (unsigned long long)staged.load(), (unsigned long long)total, (unsigned long long)zero_steps,
              (unsigned long long)links.load(), (unsigned long long)roots.load(),
              (unsigned long long)restored.load(), (unsigned long long)queries.load(), (unsigned long long)tick_busy,
              (unsigned long long)busy.load());
  return 0;
}
