// In-process transport between W virtual ranks that run on W host threads of one process: the
// Communicator of LocalReducerGroup, which runs the generic reducers (SRA / Ring / all-to-all /
// compressed broadcast) on host memory and on ONE GPU, so that their device path is testable
// without a second GPU or a c10d backend.
//
// Every rank numbers its exchange() calls. A message is matched by (exchange index, src, dst), one
// per pair and exchange, as C10dCommunicator assumes. The receiver copies the sender's bytes
// on its own stream, and waits for the copy, once both sides have posted the exchange; exchange() returns when this rank's
// receives have landed and its sends have been consumed (the reducers reuse their send buffers
// right away). All waits are host-side and bounded by the timeout; a mismatch (byte counts, a
// missing partner) or a timeout fails the whole hub, which releases every waiting rank.
#pragma once
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "communicator.h"

namespace cgx {

class LoopbackHub {
 public:
  struct Message {
    int64_t exchange;
    int src, dst;
    std::vector<uint8_t> bytes;  // host copy of what was moved
  };

  LoopbackHub(int world, int64_t timeout_ms);
  int world() const { return world_; }
  // before a collective: exchange counters, posted operations, failure and recorded messages
  void reset(bool record);
  // called by rank `rank` when its collective has returned (or thrown): peers stop waiting for it
  void finish(int rank);
  // the first failure wins; every waiting rank is released and throws
  void fail(const std::string& msg);
  bool failed() const;
  std::string failure() const;
  std::vector<Message> messages() const;  // sorted by (exchange, src, dst)

  // `cuda`: buffers are device memory; `stream` has produced the send data and is synchronised first
  void exchange(int rank, const std::vector<P2POp>& ops, bool cuda, cudaStream_t stream);
  void barrier(int rank);

 private:
  struct Posted {
    std::vector<P2POp> ops;
    std::vector<char> consumed;  // per op: a send that its receiver has copied
  };
  // wait on cv_ until pred() or failure; on timeout fail with `what`
  template <class Pred>
  void wait_for(std::unique_lock<std::mutex>& lk, Pred pred, const std::string& what);
  void throw_if_failed() const;
  void fail_locked(const std::string& msg);
  static const P2POp* find(const Posted& p, bool send, int peer, size_t* index);

  const int world_;
  const std::chrono::milliseconds timeout_;
  mutable std::mutex mu_;
  std::condition_variable cv_;
  std::vector<std::vector<Posted>> posted_;  // [rank][exchange]
  std::vector<char> done_;
  std::string failure_;
  bool record_ = false;
  std::vector<Message> messages_;
  uint64_t barrier_gen_ = 0;
  int barrier_count_ = 0;
};

class LoopbackCommunicator : public Communicator {
 public:
  LoopbackCommunicator(LoopbackHub* hub, int rank, bool cuda) : hub_(hub), rank_(rank), cuda_(cuda) {}
  int rank() const override { return rank_; }
  int size() const override { return hub_->world(); }
  bool is_cuda() const override { return cuda_; }
  void exchange(const std::vector<P2POp>& ops, cudaStream_t stream) override {
    hub_->exchange(rank_, ops, cuda_, stream);
  }
  void barrier() override { hub_->barrier(rank_); }

 private:
  LoopbackHub* hub_;
  int rank_;
  bool cuda_;
};

}  // namespace cgx
