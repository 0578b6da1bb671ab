// Batcher: the trigger / index bookkeeping of the Go sidecar's BatchHandler as a deterministic state machine
// (pkg/batcher/handler.go:157-199).  A fired batch runs as one b200_batch_predict call.
#pragma once
#include <deque>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------------
// Trigger state machine.  Time is supplied by the caller (microseconds) so the logic is testable and the
// host language keeps its own concurrency (goroutines + channels in Go, asyncio in Python):
//   add()  == the `case req := <-handler.channelIn` arm      (handler.go:162-177)
//   tick() == the check after every select iteration          (handler.go:180-186)
// A batch fires when CurrentInputLen >= MaxBatchSize (instances, not requests; the whole request is
// appended before the check, so batches may exceed the maximum) or when whole milliseconds since the first
// instance >= MaxLatency and the batch is not empty.
// ---------------------------------------------------------------------------------------------------
struct BatcherCore {
  int max_batch_size, max_latency_ms;
  long long start_us = 0;
  int current_len = 0;
  long long next_ticket = 1;
  struct Req { long long ticket; int first, count; };
  std::vector<Req> reqs;
  std::mutex mu;

  BatcherCore(int mbs, int ml) : max_batch_size(mbs <= 0 ? 32 : mbs), max_latency_ms(ml <= 0 ? 5000 : ml) {}

  long long add(long long now_us, int n_instances) {
    std::lock_guard<std::mutex> g(mu);
    if (current_len == 0) start_us = now_us;  // "if len(Instances) == 0 { Start = now }"
    Req r{next_ticket++, current_len, n_instances};
    reqs.push_back(r);
    current_len += n_instances;
    return r.ticket;
  }
  // returns the number of requests in the fired batch (0 = no trigger)
  int tick(long long now_us, long long* tickets, int* first, int* count, int cap, int* total_instances) {
    std::lock_guard<std::mutex> g(mu);
    const long long elapsed_ms = (now_us - start_us) / 1000;  // Duration.Milliseconds() truncates
    const bool fire = current_len >= max_batch_size || (elapsed_ms >= max_latency_ms && current_len > 0);
    if (!fire) return 0;
    const int n = (int)reqs.size();
    if (n > cap) return -1;
    for (int i = 0; i < n; ++i) { tickets[i] = reqs[i].ticket; first[i] = reqs[i].first; count[i] = reqs[i].count; }
    *total_instances = current_len;
    reqs.clear();
    current_len = 0;
    start_us = now_us;  // InitializeInfo(): Start = now
    return n;
  }
};

}  // namespace b200
